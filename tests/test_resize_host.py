"""CPU tests of the raw-image input side: the numpy restatement of Pillow's BILINEAR resampling (tests/resize_oracle.py)
is bit-exact against Pillow's own outputs (the SHA-256 of their bytes in tests/golden/resize_pil.npz, written by
oracle/gen_golden_resize.py), engine.resize_ratio reproduces the reference's sizes, and odtk_preprocess_resize_u8
validates its arguments and answers its size query without a GPU."""
import ctypes
import os

import numpy as np
import pytest
import torch

import resize_oracle
from retinanet_examples_b200 import _lib, engine


@pytest.fixture(scope="module")
def fixture(golden_dir):
    return np.load(os.path.join(golden_dir, "resize_pil.npz"))


def test_fixture_covers_the_cases(fixture):
    names = list(fixture["names"])
    assert str(fixture["pillow_version"])
    shapes = {n: (fixture[n + "_img"].shape[:2], tuple(fixture[n + "_dst"])) for n in names}
    assert any(d[0] < s[0] and d[1] < s[1] for s, d in shapes.values())           # downscale
    assert any(d[0] > s[0] and d[1] > s[1] for s, d in shapes.values())           # upscale
    assert any(s == d for s, d in shapes.values())                                # same size
    assert any(d[1] == 1333 and d[0] < 800 for _, d in shapes.values())          # max_size cap
    assert any(s[0] > s[1] for s, _ in shapes.values()) and any(s[0] < s[1] for s, _ in shapes.values())
    assert any(min(s) < 8 for s, _ in shapes.values())                            # tiny
    outs = [resize_oracle.fixture_output(fixture, n) for n in names]
    assert any((o == 0).any() and (o == 255).any() for o in outs)


def test_oracle_matches_pillow_bit_for_bit(fixture):
    for n in fixture["names"]:
        dh, dw = (int(v) for v in fixture[n + "_dst"])
        got = resize_oracle.resize_bilinear(fixture[n + "_img"], dh, dw)
        assert got.shape == (dh, dw, 3)
        assert resize_oracle.digest(got) == str(fixture[n + "_pil_sha256"]), n
    # the digest catches a single flipped bit
    got[0, 0, 0] ^= 1
    assert resize_oracle.digest(got) != str(fixture[n + "_pil_sha256"])


def test_resize_ratio_matches_fixture(fixture):
    resize, max_size = int(fixture["resize"]), int(fixture["max_size"])
    for n in fixture["names"]:
        h, w = fixture[n + "_img"].shape[:2]
        ratio, dh, dw = engine.resize_ratio(h, w, resize, max_size)
        assert ratio == float(fixture[n + "_ratio"]), n
        assert (dh, dw) == tuple(int(v) for v in fixture[n + "_dst"]), n
        assert resize_oracle.resize_ratio(h, w, resize, max_size) == (ratio, dh, dw)


def test_identity_axis_weights():
    lo, k = resize_oracle.coeffs(517, 517)
    assert (lo == np.arange(517)).all() and (k[:, 0] == 1 << 22).all() and (k[:, 1:] == 0).all()


def test_plan_canvas_is_the_reference_collate():
    plan = engine.ResizePlan([(480, 640), (640, 427), (333, 517), (100, 1400)], 800, 1333)
    dst = [(t.dst_h, t.dst_w) for t in plan.table]
    assert dst == [(800, 1066), (1199, 800), (800, 1242), (95, 1333)]
    assert plan.canvas == (1280, 1408)                            # max of the 128-padded sizes
    assert [t.offset for t in plan.table] == [0, 480 * 640 * 3, 480 * 640 * 3 + 640 * 427 * 3, 480 * 640 * 3 + 640 * 427 * 3 + 333 * 517 * 3]
    assert plan.nbytes == 3 * (480 * 640 + 640 * 427 + 333 * 517 + 100 * 1400)
    np.testing.assert_array_equal(plan.ratios.numpy(), np.float32([800 / 480, 800 / 427, 800 / 333, 1333 / 1400]))
    assert engine.ResizePlan([(480, 640)], 800, 1333, canvas=(896, 1152)).canvas == (896, 1152)
    with pytest.raises(ValueError):
        engine.ResizePlan([(480, 640)], 800, 1333, canvas=(768, 1152))      # too small
    with pytest.raises(ValueError):
        engine.ResizePlan([(480, 640)], 800, 1333, canvas=(896, 1100))      # not a multiple of the stride
    with pytest.raises(ValueError):
        engine.ResizePlan([(1, 4000)], 800, 1333)                            # resizes to 0 rows


def _call(table, canvas_h, canvas_w, x_bytes, y=None):
    arr = (_lib.ResizeImage * len(table))()
    for t, (off, sh, sw, dh, dw) in zip(arr, table):
        t.offset, t.src_h, t.src_w, t.dst_h, t.dst_w = off, sh, sw, dh, dw
    return _lib.lib().odtk_preprocess_resize_u8(None, x_bytes, ctypes.byref(arr), None, len(table), canvas_h, canvas_w, y,
                                                None, None, None)


def test_abi_size_query_and_validation_need_no_gpu():
    ok = [(0, 480, 640, 800, 1066), (480 * 640 * 3, 3, 5, 799, 1333)]
    xb = 480 * 640 * 3 + 45
    assert _call(ok, 896, 1408, xb) == 2 * (896 + 6) * (1408 + 8) * 8
    assert _call(ok, 896, 1408, xb - 1) == -1                                  # last image past x_bytes
    assert _call(ok, 896, 1333, xb) == -1                                       # odd canvas side
    assert _call(ok, 799, 1408, xb) == -1                                       # dst_h does not fit
    assert _call(ok, 896, 1332, xb) == -1                                       # dst_w does not fit
    for bad in ((0, 0, 640, 800, 1066), (0, 480, -1, 800, 1066), (0, 480, 640, 0, 1066), (0, 480, 640, 800, -3),
                (-1, 480, 640, 800, 1066)):
        assert _call([bad], 896, 1408, xb) == -1, bad
    assert _call(ok, 0, 1408, xb) == -1
    assert _lib.lib().odtk_preprocess_resize_u8(None, xb, None, None, 1, 896, 1408, None, None, None, None) == -1


def test_images_are_checked():
    with pytest.raises(ValueError):
        engine.preprocess_resize_u8([torch.zeros((10, 10, 3), dtype=torch.float32)], 800, 1333)
    with pytest.raises(ValueError):
        engine.preprocess_resize_u8([torch.zeros((10, 10), dtype=torch.uint8)], 800, 1333)
