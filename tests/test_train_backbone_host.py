"""CPU tests of training ResNet stages 3-4: the parameter names, shapes and order of the "layer4" / "layer3" scopes against
the reference (torchvision's ResNet registration order; ResNet18 against the reference golden's named_parameters()), the
scopes' argument checks, the new C-ABI cases' argument checks without a GPU, and the identity behind a stride-2 1x1 input
gradient (scatter to the even positions + the stride-1 1x1 == d/dx of the strided 1x1)."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from retinanet_examples_b200 import _lib, engine
from retinanet_examples_b200.model import Model, make_state_dict

RESNETS = ("ResNet18FPN", "ResNet34FPN", "ResNet50FPN", "ResNet101FPN", "ResNet152FPN")


def _reference_stage_names(backbone, levels):
    """torchvision's ResNet parameter registration order (what the reference's ResNet subclasses): per block conv1, bn1,
    conv2, bn2(, conv3, bn3), downsample.0, downsample.1 -- the conv weights of the given layers."""
    import torchvision
    net = getattr(torchvision.models, backbone[:-3].lower())(weights=None)
    names = [n for n, p in net.named_parameters() if n.split(".")[0] in ["layer%d" % (l - 1) for l in levels]]
    return [("backbones.%s.features.%s" % (backbone, n), tuple(dict(net.named_parameters())[n].shape)) for n in names
            if ".bn" not in n and not n.endswith(("downsample.1.weight", "downsample.1.bias"))]


@pytest.mark.parametrize("backbone", RESNETS)
@pytest.mark.parametrize("scope,levels", [("layer4", (5,)), ("layer3", (4, 5))])
def test_stage_scope_parameter_names_shapes_order(backbone, scope, levels):
    m = Model(backbone, classes=5)
    assert m.set_train_scope(scope) is m
    sd = make_state_dict(backbone, 5, m.num_anchors, False)
    ref = _reference_stage_names(backbone, levels)
    names = m._param_names()
    bb = m._backbone_param_names()
    assert [(n, tuple(sd[n].shape)) for n in bb] == ref
    assert names == bb + m._fpn_param_names() + m._head_param_names()
    assert not any(".bn" in n or n.endswith(".bias") for n in bb)


def test_resnet18_order_matches_the_reference_golden(golden_dir):
    names = [str(n) for n in np.load(os.path.join(golden_dir, "backbone_grads.npz"))["names"]]
    m = Model("ResNet18FPN", classes=3).set_train_scope("layer3")
    stage = [n for n in names if (".layer3." in n or ".layer4." in n) and n.endswith(".weight")]
    assert m._backbone_param_names() == stage
    assert m._param_names()[len(stage):len(stage) + 16] == [n for n in names if ".features." not in n and n.startswith("backbones")]
    assert m.set_train_scope("layer4")._backbone_param_names() == [n for n in stage if ".layer4." in n]


def test_stage_scope_argument_checks():
    for b in ("ResNeXt50_32x4dFPN", "ResNeXt101_32x8dFPN"):
        for scope in ("layer4", "layer3"):
            with pytest.raises(ValueError, match="grouped"):
                Model(b, classes=3).set_train_scope(scope)
        Model(b, classes=3).set_train_scope("fpn")
    for scope in ("layer4", "layer3"):
        with pytest.raises(ValueError, match="64 channels"):
            Model("MobileNetV2FPN", classes=3).set_train_scope(scope)
    with pytest.raises(ValueError, match="scope"):
        Model("ResNet50FPN", classes=3).set_train_scope("layer2")
    m = Model("ResNet50FPN", classes=3).set_train_scope("layer3").set_train_scope("heads")
    assert m._param_names() == m._head_param_names()


def _dense_ex(ksize=1, stride=2):
    d = engine.WgradExDesc()
    d.g, d.x, d.dw = 256, 512, 1024
    d.n, d.g_rows, d.g_width, d.g_row0, d.cout_pad = 2, 7, 11, 0, 2048
    d.x_h, d.x_width, d.cin, d.cout = 13, 21, 1024, 2048
    d.ksize, d.stride = ksize, stride
    return d


def test_dense_wgrad_and_1x1_dgrad_argument_checks_without_a_gpu():
    L = _lib.lib()
    d = _dense_ex()
    size = L.odtk_conv_wgrad_ex(ctypes.byref(d), None, 0, None)                # dense G, 1x1 stride 2: workspace query
    assert size >= 1024 * 2048 * 4
    d.row_scale = 4096
    assert L.odtk_conv_wgrad_ex(ctypes.byref(d), None, 0, None) == size
    d.row_scale = 4098
    assert L.odtk_conv_wgrad_ex(ctypes.byref(d), None, 0, None) == -1          # misaligned scale
    d = _dense_ex()
    d.g_rows = 8
    assert L.odtk_conv_wgrad_ex(ctypes.byref(d), None, 0, None) == -1          # dense G must be the output's size
    d = _dense_ex(3, 1)
    d.g_rows, d.g_width = 13, 21
    assert L.odtk_conv_wgrad_ex(ctypes.byref(d), None, 0, None) > 0
    d = _dense_ex()
    d.tile_tab, d.tab_tiles = 2048, 4
    assert L.odtk_conv_wgrad_ex(ctypes.byref(d), None, 0, None) == -3          # 1x1 stride 2 only over a dense G

    e = engine.ConvDgradDesc()
    b = e.base
    b.x, b.w, b.y = 256, 512, 1024
    b.n, b.h, b.width, b.cin, b.cout, b.ksize, b.out_mode = 1, 8, 16, 2048, 512, 1, engine.OUT_NHWC_F16
    assert L.odtk_conv2d_dgrad(ctypes.byref(e), None) == -3                   # 1x1: only the masked instance
    e.mask = 2048                                    # (a call passing every check would launch: not with fake pointers)
    b.cout = 192
    assert L.odtk_conv2d_dgrad(ctypes.byref(e), None) == -3                   # cout % 128
    b.cout, b.tile_tab, b.tab_tiles = 512, 4096, 4
    assert L.odtk_conv2d_dgrad(ctypes.byref(e), None) == -3                   # dense only

    a, c = ctypes.c_void_p(256), ctypes.c_void_p(4096)
    #                        src  dst  n  c    src (rows, width, row0, h, w)  dst (rows, width, row0)  stride
    assert L.odtk_dilate_ex_f16(a, c, 2, 256, 7, 11, 0, 7, 11, 13, 20, 0, 2, None) == -1   # 2 (w - 1) past the width
    assert L.odtk_dilate_ex_f16(a, c, 2, 256, 7, 11, 0, 7, 11, 12, 21, 0, 2, None) == -1   # 2 (h - 1) past the rows
    assert L.odtk_dilate_ex_f16(a, c, 2, 256, 7, 11, 0, 7, 11, 13, 21, 0, 3, None) == -3   # stride 1 or 2
    assert L.odtk_dilate_ex_f16(a, a, 2, 256, 7, 11, 0, 7, 11, 13, 21, 0, 2, None) == -1   # src != dst
    assert L.odtk_dilate_ex_f16(a, c, 2, 252, 7, 11, 0, 7, 11, 13, 21, 0, 2, None) == -1   # c % 8
    assert L.odtk_dilate_ex_f16(a, c, 2, 256, 64, 48, 60, 7, 11, 7, 11, 0, 1, None) == -1  # level past the source rows
    assert _lib.lib().odtk_dilate_ex_f16.argtypes == _lib.SIGNATURES["odtk_dilate_ex_f16"][1]


@pytest.mark.parametrize("h,w", [(13, 21), (16, 24), (1, 1), (2, 3)])
def test_scatter_then_1x1_is_the_stride2_input_gradient(h, w):
    """The downsample's input gradient: G at the even positions of the input geometry, then the stride-1 1x1 with the
    transposed weights of engine.pack_weight_dgrad == d/dx of the stride-2 1x1 forward, in float64."""
    g = torch.Generator().manual_seed(h * 100 + w)
    cin, cout = 128, 256
    wt = (torch.randn((cout, cin, 1, 1), generator=g) * 0.05).half().double()
    x = torch.randn((2, cin, h, w), generator=g, dtype=torch.float64, requires_grad=True)
    y = F.conv2d(x, wt, stride=2)
    gy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    ref, = torch.autograd.grad(y, x, gy)
    gd = gy.new_zeros((2, cout, h, w))
    gd[:, :, 0::2, 0::2] = gy
    wd = engine.pack_weight_dgrad(wt.float(), cout).double().view(cin, cout, 1, 1)
    torch.testing.assert_close(F.conv2d(gd, wd), ref, rtol=1e-12, atol=1e-12)
