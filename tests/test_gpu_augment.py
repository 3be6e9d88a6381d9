"""GPU tests of the training input path: odtk_resize_u8_packed and odtk_augment_u8 bit-exact against the numpy oracle
(tests/augment_oracle.py, resize_oracle.py) on seeded images and parameters; the iterator over the fixture's files
reproduces the reference's batches (tests/golden/augment_ref.npz) digest for digest and its targets exactly; the
reference's training loop runs on the iterator with the losses of oracle-built batches; a corrupt scan raises naming its
file on the next batch."""
import ctypes
import os
import random

import numpy as np
import pytest
import torch

import augment_oracle as O
import resize_oracle
from retinanet_examples_b200 import _lib, engine

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _run(images, params, canvas=None, stride=1):
    """images: uint8 [h, w, 3] numpy; params: dicts of AugmentImage fields.  Returns the GPU batch [n, 3, H, W] (numpy)
    and the oracle's."""
    n = len(images)
    tab = (_lib.AugmentImage * n)()
    offs, off = [], 0
    for im in images:
        offs.append(off)
        off += im.size
    x = torch.from_numpy(np.concatenate([im.reshape(-1) for im in images])).to(DEV)
    ref = []
    for t, im, o, p in zip(tab, images, offs, params):
        t.offset, t.h, t.w = o, im.shape[0], im.shape[1]
        for k, v in p.items():
            setattr(t, k, v)
        f = p.get("flags", 0)
        ref.append(O.normalize(O.augment(im, p.get("rot", 0), bool(p.get("expand", 0)), bool(p.get("flip", 0)),
                                         p.get("brightness") if f & 1 else None, p.get("contrast") if f & 2 else None,
                                         p.get("hue_shift", 0) if f & 4 else None, p.get("saturation") if f & 8 else None)))
    want = O.collate(ref, stride)
    if canvas is not None:
        w2 = np.zeros((n, 3) + canvas, np.float32)
        w2[:, :, :want.shape[2], :want.shape[3]] = want
        want = w2
    tab_dev = torch.frombuffer(bytearray(bytes(tab)), dtype=torch.uint8).to(DEV)
    got = engine.augment_launch(x, tab, tab_dev, want.shape[2:])
    assert got.is_contiguous(memory_format=torch.channels_last)
    return got.cpu().numpy(), want


def _factor(rng, large):
    return float(rng.choice([0.0, rng.uniform(0, 1), rng.uniform(1, 3), 1.0])) if large else float(rng.normal(1, 0.002))


def test_every_rotation_flip_expand_and_adjustment():
    rng = np.random.default_rng(0)
    sizes = [(5, 8), (8, 5), (7, 7), (1, 9), (9, 1), (6, 11), (11, 6), (1, 1), (13, 20)]
    for flags in (0, 1, 2, 4, 8, 15):
        for large in (False, True):
            images, params = [], []
            for h, w in sizes:
                for rot in range(4):
                    for flip in (0, 1):
                        for expand in (0, 1):
                            images.append(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
                            params.append(dict(rot=rot, flip=flip, expand=expand, flags=flags,
                                               brightness=_factor(rng, large), contrast=_factor(rng, large),
                                               saturation=_factor(rng, large), hue_shift=int(rng.integers(0, 256))))
            got, want = _run(images, params)
            assert np.array_equal(got, want), (flags, large)


def test_ragged_batch_canvas_zeros_and_rotation_fill_contrast():
    rng = np.random.default_rng(1)
    images = [rng.integers(0, 256, s + (3,), dtype=np.uint8) for s in ((37, 53), (61, 29), (20, 90), (64, 64))]
    params = [dict(rot=1, flags=2, contrast=2.5), dict(rot=3, flip=1, flags=15, brightness=1.3, contrast=0.4,
                                                       saturation=1.9, hue_shift=200),
              dict(rot=1, flags=3, brightness=0.7, contrast=3.0), dict(rot=2, flags=6, contrast=0.0, hue_shift=1)]
    got, want = _run(images, params, canvas=(128, 160), stride=32)
    assert np.array_equal(got, want)
    assert (got[0, :, 37:, :] == 0).all() and (got[0, :, :, 53:] == 0).all()


def test_all_colours_through_hue():
    c = np.arange(1 << 24, dtype=np.uint32)
    img = np.stack([(c >> 16) & 255, (c >> 8) & 255, c & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    for shift in (0, 129):
        got, want = _run([img], [dict(flags=4, hue_shift=shift)])
        assert np.array_equal(got, want), shift


def test_resize_u8_packed_matches_pillow_oracle():
    rng = np.random.default_rng(2)
    shapes = [((37, 53), (96, 137)), ((480, 640), (800, 1066)), ((61, 29), (20, 9)), ((300, 300), (31, 31)), ((5, 3), (5, 3))]
    images = [rng.integers(0, 256, s + (3,), dtype=np.uint8) for s, _ in shapes]
    tab = (_lib.ResizeImage * len(images))()
    out_off = torch.empty(len(images), dtype=torch.int64)
    so = do = 0
    for k, (t, im, (_, (dh, dw))) in enumerate(zip(tab, images, shapes)):
        t.offset, t.src_h, t.src_w, t.dst_h, t.dst_w = so, im.shape[0], im.shape[1], dh, dw
        out_off[k] = do
        so += im.size
        do += dh * dw * 3
    x = torch.from_numpy(np.concatenate([im.reshape(-1) for im in images])).to(DEV)
    tab_dev = torch.frombuffer(bytearray(bytes(tab)), dtype=torch.uint8).to(DEV)
    assert engine.resize_u8_launch(None, x.numel(), tab, None, out_off, None, None) == do
    y = torch.full((do,), 7, dtype=torch.uint8, device=DEV)
    engine.resize_u8_launch(x, x.numel(), tab, tab_dev, out_off, out_off.to(DEV), y)
    y = y.cpu().numpy()
    for k, (im, (_, (dh, dw))) in enumerate(zip(images, shapes)):
        o = int(out_off[k])
        assert np.array_equal(y[o:o + dh * dw * 3].reshape(dh, dw, 3), resize_oracle.resize_bilinear(im, dh, dw)), k


@pytest.fixture(scope="module")
def fixture(golden_dir):
    return np.load(os.path.join(golden_dir, "augment_ref.npz"))


def _pillow():
    try:
        import PIL  # noqa: F401
        return True
    except ImportError:
        return False


def test_iterator_reproduces_reference(fixture, tmp_path):
    if not _pillow():
        pytest.skip("Pillow is not installed: the progressive fixture file has no host decoder")
    for ci, cfg in enumerate(O.fixture_configs(fixture)):
        ann = O.fixture_dir(fixture, str(tmp_path), cfg["rotated"])
        it = O.make_iterator(cfg, str(tmp_path), ann, random.Random(cfg["seed"]))
        for bi, idx in enumerate(cfg["batches"]):
            out = it.batch(idx)
            data = out[0]
            assert data.is_contiguous(memory_format=torch.channels_last)
            assert data.contiguous(memory_format=torch.channels_last).data_ptr() == data.data_ptr()
            nchw = data.contiguous().cpu().numpy()
            assert tuple(nchw.shape) == tuple(fixture["cfg%d_b%d_shape" % (ci, bi)]), cfg["name"]
            assert O.sha256(nchw) == cfg["sha256"][bi], (cfg["name"], bi)
            if cfg["training"]:
                assert torch.equal(out[1].cpu(), torch.from_numpy(fixture["cfg%d_b%d_target" % (ci, bi)])), (cfg["name"], bi)
            else:
                assert torch.equal(out[1].cpu(), torch.from_numpy(fixture["cfg%d_b%d_ids" % (ci, bi)]))
                assert torch.equal(out[2].cpu(), torch.from_numpy(fixture["cfg%d_b%d_ratios" % (ci, bi)]))
        it._check_pending()


def test_iteration_and_length(fixture, tmp_path):
    cfg = O.fixture_configs(fixture)[0]
    ann = O.fixture_dir(fixture, str(tmp_path), False)
    it = O.make_iterator(cfg, str(tmp_path), ann, random.Random(0))
    batches = list(it)
    assert len(batches) == len(it) == 2                 # 12 images, batch 8, the last partial batch kept
    assert [b[0].shape[0] for b in batches] == [8, 4]


def test_corrupt_scan_raises_on_next_batch(fixture, tmp_path, golden_dir):
    cfg = dict(O.fixture_configs(fixture)[0])
    ann = O.fixture_dir(fixture, str(tmp_path), False)
    bad = np.load(os.path.join(golden_dir, "jpeg_pil.npz"))["truncated_jpeg"].tobytes()
    with open(os.path.join(str(tmp_path), "a_420_37x53.jpg"), "wb") as f:
        f.write(bad)
    it = O.make_iterator(cfg, str(tmp_path), ann, random.Random(0))
    it.batch([0, 1])                                    # the decode status is read one batch late
    with pytest.raises(RuntimeError, match="a_420_37x53.jpg"):
        it.batch([2, 3])


LARGE_AUG = dict(augment_brightness=0.8, augment_contrast=0.9, augment_hue=0.4, augment_saturation=1.2)


def _train(feed, epochs):
    """The reference's training loop (odtk/train.py:96-123: zero_grad, model([data.contiguous(channels_last), target]),
    GradScaler-scaled backward, step, update) on a ResNet18FPN in the heads scope; returns each step's two losses."""
    from retinanet_examples_b200.model import Model, make_state_dict
    m = Model("ResNet18FPN", classes=3).load_state_dict(make_state_dict("ResNet18FPN", 3, 9, False, seed=6)).cuda(0)
    m.train()
    opt = torch.optim.SGD(m.parameters(), lr=0.01, weight_decay=1e-4, momentum=0.9)
    scaler = torch.amp.GradScaler("cuda")
    losses = []
    for _ in range(epochs):
        for data, target in feed():
            opt.zero_grad()
            cls_loss, box_loss = m([data.contiguous(memory_format=torch.channels_last), target])
            del data
            scaler.scale(cls_loss + box_loss).backward()
            scaler.step(opt)
            scaler.update()
            losses.append((float(cls_loss.detach()), float(box_loss.detach())))
    return losses


def test_reference_training_loop_on_the_iterator(fixture, tmp_path):
    """The loop runs unmodified on the iterator, and its losses equal, bit for bit, the same loop fed with batches the
    numpy oracle built from the same draws (two epochs, batch 4, stride 128, rotation and large augment values)."""
    if not _pillow():
        pytest.skip("Pillow is not installed: the progressive fixture file has no host decoder")
    from retinanet_examples_b200 import data as D
    d = str(tmp_path)
    ann = O.fixture_dir(fixture, d, False)
    make = lambda: D.DataIterator(d, [96, 160], 256, 4, 128, 1, ann, training=True, rotate_augment=True,   # noqa: E731
                                  rng=random.Random(11), **LARGE_AUG)
    it = make()
    got = _train(lambda: it, 2)
    ref_it = make()

    def oracle_feed():
        n = len(ref_it.ids)
        for i in range(0, n, 4):
            x, t = O.oracle_batch(ref_it, list(range(i, min(i + 4, n))))
            yield torch.from_numpy(x).to(DEV), t.to(DEV)

    want = _train(oracle_feed, 2)
    assert len(got) == 6 and got == want
