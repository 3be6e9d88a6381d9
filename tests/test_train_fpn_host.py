"""CPU tests of FPN training's host side: parameter names / shapes / order of the "fpn" scope, the scope's argument checks,
the new C-ABI entry points' argument checks and workspace query, and the identity behind pyramid7's input gradient
(dilation + the stride-1 rotated-weight convolution == the input gradient of a stride-2 pad-1 3x3)."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from retinanet_examples_b200 import _lib, engine
from retinanet_examples_b200.model import Model, make_state_dict

CHANNELS = {"ResNet18FPN": (128, 256, 512), "ResNet34FPN": (128, 256, 512), "ResNet50FPN": (512, 1024, 2048),
            "ResNet101FPN": (512, 1024, 2048), "ResNeXt50_32x4dFPN": (512, 1024, 2048)}


def _reference_fpn(channels):
    """The reference FPN's own convolutions (odtk/backbones/fpn.py:26-33), in its registration order."""
    m = torch.nn.Module()
    m.lateral3 = torch.nn.Conv2d(channels[0], 256, 1)
    m.lateral4 = torch.nn.Conv2d(channels[1], 256, 1)
    m.lateral5 = torch.nn.Conv2d(channels[2], 256, 1)
    m.pyramid6 = torch.nn.Conv2d(channels[2], 256, 3, stride=2, padding=1)
    m.pyramid7 = torch.nn.Conv2d(256, 256, 3, stride=2, padding=1)
    m.smooth3 = torch.nn.Conv2d(256, 256, 3, padding=1)
    m.smooth4 = torch.nn.Conv2d(256, 256, 3, padding=1)
    m.smooth5 = torch.nn.Conv2d(256, 256, 3, padding=1)
    return m


@pytest.mark.parametrize("backbone", sorted(CHANNELS))
def test_fpn_scope_parameter_names_shapes_order(backbone):
    m = Model(backbone, classes=5)
    assert m.set_train_scope("fpn") is m
    sd = make_state_dict(backbone, 5, m.num_anchors, False)
    ref = [("backbones.%s.%s" % (backbone, n), tuple(p.shape)) for n, p in _reference_fpn(CHANNELS[backbone]).named_parameters()]
    ref += [(n, tuple(sd[n].shape)) for n in m._head_param_names()]
    assert [(n, tuple(sd[n].shape)) for n in m._param_names()] == ref
    assert len(m._fpn_param_names()) == 16


def test_default_scope_is_the_heads():
    m = Model("ResNet50FPN", classes=3)
    assert m.train_scope == "heads"
    assert m._param_names() == m._head_param_names()
    m.set_train_scope("fpn").set_train_scope("heads")
    assert m._param_names() == m._head_param_names()


def test_scope_argument_checks():
    with pytest.raises(ValueError, match="64 channels"):
        Model("MobileNetV2FPN", classes=3).set_train_scope("fpn")
    Model("MobileNetV2FPN", classes=3).set_train_scope("heads")
    with pytest.raises(ValueError, match="scope"):
        Model("ResNet18FPN", classes=3).set_train_scope("backbone")


def test_new_signatures_resolve():
    L = _lib.lib()
    for name in ("odtk_conv_wgrad_ex", "odtk_pool_add_f16", "odtk_dilate_f16"):
        assert name in _lib.SIGNATURES
        assert getattr(L, name).argtypes == _lib.SIGNATURES[name][1]


def _valid_ex(ksize=1, stride=1):
    d = engine.WgradExDesc()
    d.g, d.x, d.dw, d.tile_tab = 256, 512, 1024, 2048
    d.n, d.g_rows, d.g_width, d.g_row0, d.cout_pad = 2, 64, 48, 40, 256
    d.x_h, d.x_width, d.cin, d.cout = 10, 12, 512, 256
    d.ksize, d.stride, d.tab_tiles = ksize, stride, 2
    return d


def test_wgrad_ex_argument_checks_without_a_gpu():
    L = _lib.lib()
    assert L.odtk_conv_wgrad_ex(None, None, 0, None) == -1
    for ks, st in ((1, 1), (3, 1), (3, 2)):
        d = _valid_ex(ks, st)
        size = L.odtk_conv_wgrad_ex(ctypes.byref(d), None, 0, None)             # workspace query: no CUDA call
        assert size >= ks * ks * 512 * 256 * 4, (ks, st)
        assert L.odtk_conv_wgrad_ex(ctypes.byref(d), ctypes.c_void_p(4096), size - 1, None) == -2
    for field in ("g", "x", "dw", "tile_tab"):                                  # null pointers
        d = _valid_ex()
        setattr(d, field, None)
        assert L.odtk_conv_wgrad_ex(ctypes.byref(d), None, 0, None) == -1, field
    for ks, st in ((1, 2), (3, 3), (5, 1), (2, 1), (0, 1)):                     # only 1x1 s1, 3x3 s1, 3x3 s2
        assert L.odtk_conv_wgrad_ex(ctypes.byref(_valid_ex(ks, st)), None, 0, None) == -3, (ks, st)
    d = _valid_ex()
    d.cin = 192
    assert L.odtk_conv_wgrad_ex(ctypes.byref(d), None, 0, None) == -3          # 128-channel N tiles
    d = _valid_ex()
    d.cout, d.cout_pad = 80, 96
    assert L.odtk_conv_wgrad_ex(ctypes.byref(d), None, 0, None) == -3          # 64-channel G boxes
    d = _valid_ex()
    d.cout = 320
    assert L.odtk_conv_wgrad_ex(ctypes.byref(d), None, 0, None) == -1          # cout > cout_pad
    d = _valid_ex()
    d.g_row0 = 60                                                               # 10-row level runs past the atlas
    assert L.odtk_conv_wgrad_ex(ctypes.byref(d), None, 0, None) == -1
    d = _valid_ex()
    d.x_width = 60                                                              # level wider than the atlas
    assert L.odtk_conv_wgrad_ex(ctypes.byref(d), None, 0, None) == -1
    d = _valid_ex()
    d.tab_tiles = 0
    assert L.odtk_conv_wgrad_ex(ctypes.byref(d), None, 0, None) == -1
    d = _valid_ex()
    d.x = 520                                                                   # misaligned
    assert L.odtk_conv_wgrad_ex(ctypes.byref(d), None, 0, None) == -1


def test_small_kernel_argument_checks_without_a_gpu():
    L = _lib.lib()
    a, b = ctypes.c_void_p(256), ctypes.c_void_p(4096)
    #                       src   dst  n  rows width c   src (row0, h, w)   dst (row0, h, w)  pool
    assert L.odtk_pool_add_f16(None, b, 1, 64, 48, 256, 0, 32, 48, 40, 16, 24, 2, None) == -1
    assert L.odtk_pool_add_f16(a, None, 1, 64, 48, 256, 0, 32, 48, 40, 16, 24, 2, None) == -1
    assert L.odtk_pool_add_f16(a, b, 1, 64, 48, 256, 0, 32, 48, 40, 16, 24, 3, None) == -3     # pool 1 or 2
    assert L.odtk_pool_add_f16(a, b, 1, 64, 48, 252, 0, 32, 48, 40, 16, 24, 2, None) == -1     # c % 8
    assert L.odtk_pool_add_f16(a, b, 1, 64, 48, 256, 0, 32, 48, 50, 16, 24, 2, None) == -1     # dst past the rows
    assert L.odtk_pool_add_f16(a, b, 1, 64, 48, 256, 0, 32, 48, 40, 16, 50, 2, None) == -1     # dst wider than the atlas
    assert L.odtk_pool_add_f16(a, a, 1, 64, 48, 256, 0, 32, 48, 20, 16, 24, 2, None) == -1     # in place, overlapping rows
    assert L.odtk_dilate_f16(None, b, 1, 64, 48, 256, 40, 8, 12, 0, None) == -1
    assert L.odtk_dilate_f16(a, b, 1, 64, 48, 252, 40, 8, 12, 0, None) == -1                     # c % 8
    assert L.odtk_dilate_f16(a, b, 1, 64, 48, 256, 40, 8, 25, 0, None) == -1                     # 2 w > width
    assert L.odtk_dilate_f16(a, b, 1, 64, 48, 256, 40, 8, 12, 50, None) == -1                    # 2 h past the rows


@pytest.mark.parametrize("h6,w6", [(13, 20), (25, 40), (7, 10), (8, 10), (1, 1), (2, 3)])
def test_dilation_then_stride1_dgrad_is_the_stride2_input_gradient(h6, w6):
    """pyramid7's input gradient: G scattered to the even positions of P6's geometry, convolved (stride 1, pad 1) with
    the rotated weights of engine.pack_weight_dgrad == d/dx of the stride-2 pad-1 3x3 forward, in float64."""
    g = torch.Generator().manual_seed(h6 * 100 + w6)
    c = 128
    w = (torch.randn((c, c, 3, 3), generator=g) * 0.05).half().double()
    x = torch.randn((2, c, h6, w6), generator=g, dtype=torch.float64, requires_grad=True)
    y = F.conv2d(x, w, stride=2, padding=1)
    h7, w7 = y.shape[2:]
    assert (h7, w7) == ((h6 - 1) // 2 + 1, (w6 - 1) // 2 + 1) and 2 * (h7 - 1) <= h6 - 1
    gy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    ref, = torch.autograd.grad(y, x, gy)
    gd = gy.new_zeros((2, c, h6, w6))
    gd[:, :, 0::2, 0::2] = gy
    wd = engine.pack_weight_dgrad(w.float(), c).double().view(c, 3, 3, c).permute(0, 3, 1, 2)
    torch.testing.assert_close(F.conv2d(gd, wd, padding=1), ref, rtol=1e-12, atol=1e-12)
