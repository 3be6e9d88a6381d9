"""CPU tests of the argument checks of the convolution entry points (odtk_conv2d, odtk_conv2d_dgrad, odtk_conv2d_s8,
odtk_conv2d_s8_ex, odtk_conv2d_f32, odtk_stem_conv).  Each case starts from a valid descriptor with fake, aligned device
pointers and changes one field.  Every check runs before any CUDA call, so without a GPU a descriptor that passes them
returns ODTK_E_CUDA; the file is skipped when a device is visible, so that the fake pointers never reach a launch."""
import ctypes

import pytest
import torch

from retinanet_examples_b200 import _lib, engine

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="fake device pointers: run without a visible GPU")

OK, INVALID, UNSUPPORTED = -4, -1, -3      # OK: passes every check, then ODTK_E_CUDA from the first CUDA call
P = 1 << 20                                # a fake 16-byte aligned device address


def _fill(d, fields):
    for k, v in fields.items():
        obj = d
        *path, last = k.split(".")
        for p in path:
            obj = getattr(obj, p)
        assert last in {f for f, _ in obj._fields_}, k
        setattr(obj, last, v)
    return d


F16 = dict(x=P, w=2 * P, y=3 * P, n=1, h=8, width=8, cin=64, cout=64, ksize=3, out_mode=engine.OUT_NHWC_F16)
S8 = {"base." + k: v for k, v in dict(x=P, w=2 * P, alpha=4 * P, y=3 * P, n=1, h=8, width=8, cin=128, cout=64, ksize=3,
                                      out_mode=engine.OUT_NHWC_S8, inv_out_scale=1.0).items()}
F32 = dict(x=P, w_hi=2 * P, w_lo=5 * P, y=3 * P, n=1, h=8, width=8, cin=32, cout=64, ksize=3, out_mode=engine.OUT_NHWC_F32)


def _conv2d(change):
    return _lib.lib().odtk_conv2d(ctypes.byref(_fill(engine.ConvDesc(), {**F16, **change})), None)


def _dgrad(change):
    d = engine.ConvDgradDesc()
    _fill(d, {"base." + k: v for k, v in F16.items()})
    d.mask = 6 * P
    _fill(d, {k if k == "mask" else "base." + k: v for k, v in change.items()})
    return _lib.lib().odtk_conv2d_dgrad(ctypes.byref(d), None)


def _s8(change):
    d = _fill(engine.ConvS8ExDesc(), {**S8, **change})
    return _lib.lib().odtk_conv2d_s8(ctypes.byref(d.base), None)


def _s8_ex(change):
    return _lib.lib().odtk_conv2d_s8_ex(ctypes.byref(_fill(engine.ConvS8ExDesc(), {**S8, **change})), None)


def _f32(change):
    return _lib.lib().odtk_conv2d_f32(ctypes.byref(_fill(engine.ConvF32Desc(), {**F32, **change})), None)


def _stem(change):
    a = {**dict(xp=P, w=2 * P, bias=4 * P, y=3 * P, n=1, h=64, width=64, cout=64, relu=1), **change}
    return _lib.lib().odtk_stem_conv(a["xp"], a["w"], a["bias"], a["y"], a["n"], a["h"], a["width"], a["cout"], a["relu"], None)


CASES = {
    _conv2d: [
        ({}, OK), (dict(ksize=1), OK), (dict(x=None), INVALID), (dict(w=None), INVALID), (dict(y=None), INVALID),
        (dict(n=0), INVALID), (dict(h=0), INVALID), (dict(width=-1), INVALID), (dict(cin=0), INVALID), (dict(cout=0), INVALID),
        (dict(ksize=5), UNSUPPORTED), (dict(ksize=7), UNSUPPORTED), (dict(cin=48), UNSUPPORTED), (dict(cin=128), OK),
        (dict(groups=32), OK), (dict(groups=3), UNSUPPORTED), (dict(groups=2, cout=128), UNSUPPORTED),
        (dict(groups=2, ksize=1), UNSUPPORTED), (dict(groups=2, residual=4 * P), UNSUPPORTED),
        (dict(groups=2, out_mode=engine.OUT_NCHW_F32), UNSUPPORTED),
        (dict(out_mode=engine.OUT_NCHW_F32), OK), (dict(out_mode=engine.OUT_NCHW_F32_SIGMOID), OK),
        (dict(out_mode=-1), INVALID), (dict(out_mode=engine.OUT_NHWC_S8), INVALID), (dict(out_mode=engine.OUT_NHWC_F32), INVALID),
        (dict(out_mode=engine.OUT_CANDIDATES), INVALID),
        (dict(relu=1), OK), (dict(relu=2), OK), (dict(relu=2, out_mode=engine.OUT_NCHW_F32), UNSUPPORTED),
        (dict(cout=24), UNSUPPORTED), (dict(cout=24, out_mode=engine.OUT_NCHW_F32), OK),
        (dict(residual=4 * P), OK), (dict(residual=4 * P + 4), OK), (dict(residual=4 * P + 2), INVALID),
        (dict(upsample=4 * P + 2), INVALID), (dict(residual=4 * P, out_mode=engine.OUT_NCHW_F32), UNSUPPORTED),
        (dict(upsample=4 * P, out_mode=engine.OUT_NCHW_F32), UNSUPPORTED),
        (dict(n=1 << 16, h=1 << 8, width=1 << 8), UNSUPPORTED),
        (dict(x=P + 8), INVALID), (dict(w=2 * P + 8), INVALID), (dict(y=3 * P + 8), INVALID),
        (dict(y=3 * P + 8, out_mode=engine.OUT_CANDIDATES), INVALID),
    ],
    _dgrad: [
        ({}, OK), (dict(ksize=1), UNSUPPORTED), (dict(stride=2), UNSUPPORTED), (dict(relu=1), UNSUPPORTED),
        (dict(out_mode=engine.OUT_NCHW_F32), UNSUPPORTED), (dict(groups=2), UNSUPPORTED), (dict(upsample=4 * P), UNSUPPORTED),
        (dict(x_rows=16), UNSUPPORTED), (dict(x_width=16), UNSUPPORTED), (dict(y_rows=16), UNSUPPORTED),
        (dict(y_row_off=8), UNSUPPORTED), (dict(y_width=16), UNSUPPORTED), (dict(mask=6 * P + 2), INVALID), (dict(mask=None), OK),
        (dict(residual=4 * P), OK), (dict(cin=32), UNSUPPORTED), (dict(n=0), INVALID),
    ],
    _s8: [
        ({}, OK), (dict(**{"base.ksize": 1}), OK), (dict(**{"base.alpha": None}), INVALID), (dict(**{"base.x": None}), INVALID),
        (dict(**{"base.cin": 64}), UNSUPPORTED), (dict(**{"base.cin": 256}), OK), (dict(**{"base.ksize": 5}), UNSUPPORTED),
        (dict(**{"base.relu": 1}), OK), (dict(**{"base.relu": 2}), UNSUPPORTED), (dict(**{"base.relu": -1}), UNSUPPORTED),
        (dict(**{"base.out_mode": engine.OUT_NHWC_F16}), INVALID), (dict(**{"base.out_mode": engine.OUT_NHWC_F32}), INVALID),
        (dict(**{"base.out_mode": engine.OUT_NCHW_F32}), OK), (dict(**{"base.cout": 24}), UNSUPPORTED),
        (dict(**{"base.cout": 24, "base.out_mode": engine.OUT_NCHW_F32}), OK), (dict(**{"base.y": 3 * P + 8}), INVALID),
        (dict(**{"base.tile_tab": 7 * P, "base.tab_tiles": 4}), OK), (dict(**{"base.tile_tab": 7 * P}), INVALID),
        (dict(**{"base.tile_tab": 7 * P, "base.tab_tiles": 4, "base.ksize": 1}), UNSUPPORTED),
        (dict(**{"base.x_rows": 16}), OK), (dict(**{"base.x_rows": 16, "base.ksize": 1}), UNSUPPORTED),
        (dict(**{"base.x_rows": 16, "base.tile_tab": 7 * P, "base.tab_tiles": 4}), INVALID),
    ],
    _s8_ex: [
        ({}, OK), (dict(stride=2), OK), (dict(stride=2, **{"base.h": 7}), OK), (dict(stride=3), UNSUPPORTED),
        (dict(residual=4 * P), OK), (dict(residual=4 * P + 2), OK), (dict(residual=4 * P + 1), INVALID),
        (dict(upsample=4 * P + 1), INVALID), (dict(upsample=4 * P, stride=2), UNSUPPORTED),
        (dict(upsample=4 * P, **{"base.h": 7}), INVALID), (dict(residual=4 * P, **{"base.out_mode": engine.OUT_NCHW_F32}), UNSUPPORTED),
        (dict(y_rows=16), OK), (dict(y_rows=16, **{"base.out_mode": engine.OUT_NCHW_F32}), UNSUPPORTED),
        (dict(y_rows=16, **{"base.ksize": 1}), UNSUPPORTED), (dict(residual=4 * P, **{"base.x_rows": 16}), UNSUPPORTED),
        (dict(stride=2, **{"base.tile_tab": 7 * P, "base.tab_tiles": 4}), INVALID),
        (dict(y_width=16, **{"base.tile_tab": 7 * P, "base.tab_tiles": 4}), INVALID),
    ],
    _f32: [
        ({}, OK), (dict(ksize=1), OK), (dict(w_lo=None), INVALID), (dict(w_hi=None), INVALID), (dict(w_lo=5 * P + 8), INVALID),
        (dict(cin=48), UNSUPPORTED), (dict(cin=64), OK), (dict(ksize=5), UNSUPPORTED),
        (dict(ksize=7, cin=3, stride=2), OK), (dict(ksize=7, cin=3), UNSUPPORTED), (dict(ksize=7, cin=4, stride=2), UNSUPPORTED),
        (dict(ksize=7, cin=3, stride=2, residual=4 * P), UNSUPPORTED), (dict(stride=2), OK), (dict(stride=4), UNSUPPORTED),
        (dict(relu=1), OK), (dict(relu=2), UNSUPPORTED), (dict(cout=3), UNSUPPORTED), (dict(cout=3, out_mode=engine.OUT_NCHW_F32), OK),
        (dict(out_mode=engine.OUT_NHWC_F16), INVALID), (dict(out_mode=engine.OUT_NHWC_S8), INVALID),
        (dict(residual=4 * P), OK), (dict(residual=4 * P + 8), OK), (dict(residual=4 * P + 4), INVALID),
        (dict(upsample=4 * P, stride=2), UNSUPPORTED), (dict(upsample=4 * P, h=7), INVALID),
        (dict(upsample=4 * P, out_mode=engine.OUT_NCHW_F32), UNSUPPORTED), (dict(y_rows=16), OK),
        (dict(y_rows=16, out_mode=engine.OUT_NCHW_F32), UNSUPPORTED), (dict(tile_tab=7 * P, tab_tiles=4), OK),
        (dict(tile_tab=7 * P, tab_tiles=0), INVALID), (dict(tile_tab=7 * P, tab_tiles=4, stride=2), INVALID),
        (dict(x_width=16, ksize=1), UNSUPPORTED), (dict(n=1 << 16, h=1 << 8, width=1 << 8), UNSUPPORTED),
    ],
    _stem: [
        ({}, OK), (dict(cout=128), OK), (dict(xp=None), INVALID), (dict(y=None), INVALID), (dict(n=0), INVALID),
        (dict(h=63), UNSUPPORTED), (dict(width=63), UNSUPPORTED), (dict(cout=24), UNSUPPORTED), (dict(cout=144), UNSUPPORTED),
        (dict(w=2 * P + 8), INVALID), (dict(y=3 * P + 4), INVALID),
    ],
}


@pytest.mark.parametrize("entry,change,expected", [(e, c, r) for e, cases in CASES.items() for c, r in cases],
                         ids=["%s-%s" % (e.__name__[1:], "-".join("%s=%s" % kv for kv in c.items()) or "valid")
                              for e, cases in CASES.items() for c, _ in cases])
def test_conv_argument_checks(entry, change, expected):
    assert entry(change) == expected


def test_null_descriptors_are_invalid():
    L = _lib.lib()
    for name in ("odtk_conv2d", "odtk_conv2d_dgrad", "odtk_conv2d_s8", "odtk_conv2d_s8_ex", "odtk_conv2d_f32"):
        assert getattr(L, name)(None, None) == INVALID, name
