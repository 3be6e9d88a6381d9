"""CPU tests of the head-training host side: parameter names / shapes / order, the new C-ABI entry points' argument
checks and workspace query, and the input-gradient weight repacking (engine.pack_weight_dgrad)."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from retinanet_examples_b200 import _lib, engine
from retinanet_examples_b200.model import Model, make_state_dict


def _reference_heads(classes, num_anchors, rotated):
    """The reference's head modules (odtk/model.py:57-68): 4 x (conv 3x3 256, ReLU) + a final conv 3x3."""
    def make_head(out):
        layers = []
        for _ in range(4):
            layers += [torch.nn.Conv2d(256, 256, 3, padding=1), torch.nn.ReLU()]
        layers += [torch.nn.Conv2d(256, out, 3, padding=1)]
        return torch.nn.Sequential(*layers)
    m = torch.nn.Module()
    m.cls_head = make_head(classes * num_anchors)
    m.box_head = make_head((6 if rotated else 4) * num_anchors)
    return m


@pytest.mark.parametrize("rotated", [False, True])
def test_parameter_names_shapes_order_match_reference_heads(rotated):
    m = Model("ResNet18FPN", classes=5, rotated_bbox=rotated)
    sd = make_state_dict("ResNet18FPN", 5, m.num_anchors, rotated)
    ref = [(n, tuple(p.shape)) for n, p in _reference_heads(5, m.num_anchors, rotated).named_parameters()]
    ours = [(n, tuple(sd[n].shape)) for n in m._head_param_names()]
    assert ours == ref


def test_parameters_need_cuda():
    m = Model("ResNet18FPN", classes=3).load_state_dict(make_state_dict("ResNet18FPN", 3, 9, False))
    with pytest.raises(RuntimeError, match="cuda"):
        list(m.parameters())


def test_new_signatures_resolve():
    L = _lib.lib()
    for name in ("odtk_conv_wgrad", "odtk_grad_to_atlas", "odtk_conv2d_dgrad"):
        assert name in _lib.SIGNATURES
        assert getattr(L, name).argtypes == _lib.SIGNATURES[name][1]


def test_abi_argument_checks_without_a_gpu():
    L = _lib.lib()
    assert L.odtk_conv_wgrad(None, None, 0, None) == -1
    d = engine.WgradDesc()
    assert L.odtk_conv_wgrad(ctypes.byref(d), None, 0, None) == -1            # null pointers
    d.g, d.x, d.dw = 256, 512, 1024
    d.n, d.h, d.width, d.cin, d.cout, d.cout_pad = 1, 8, 16, 256, 36, 64
    size = L.odtk_conv_wgrad(ctypes.byref(d), None, 0, None)                   # workspace query: no CUDA call
    assert size >= 9 * 256 * 64 * 4
    assert L.odtk_conv_wgrad(ctypes.byref(d), ctypes.c_void_p(4096), size - 1, None) == -2
    d.cin = 192
    assert L.odtk_conv_wgrad(ctypes.byref(d), None, 0, None) == -3            # 128-channel N tiles
    d.cin, d.cout_pad = 256, 96
    assert L.odtk_conv_wgrad(ctypes.byref(d), None, 0, None) == -3            # 64-channel G boxes
    d.cout, d.cout_pad = 80, 64
    assert L.odtk_conv_wgrad(ctypes.byref(d), None, 0, None) == -1            # cout > cout_pad

    assert L.odtk_grad_to_atlas(1, 1, None, 36, None, None, 8, 16, 64, None) == -1
    lv = (engine.GradLevel * 1)()
    lv[0].grad, lv[0].height, lv[0].width, lv[0].row0 = 256, 8, 16, 0
    assert L.odtk_grad_to_atlas(1, 1, ctypes.cast(lv, ctypes.c_void_p), 36, None, None, 8, 16, 64, None) == -1
    assert L.odtk_grad_to_atlas(1, 1, ctypes.cast(lv, ctypes.c_void_p), 80, None, ctypes.c_void_p(256), 8, 16, 64, None) == -1
    lv[0].row0 = 1                                                              # level runs past the atlas rows
    assert L.odtk_grad_to_atlas(1, 1, ctypes.cast(lv, ctypes.c_void_p), 36, None, ctypes.c_void_p(256), 8, 16, 64, None) == -1
    assert L.odtk_grad_to_atlas(1, 9, ctypes.cast(lv, ctypes.c_void_p), 36, None, ctypes.c_void_p(256), 8, 16, 64, None) == -3
    lv[0].row0 = 0
    assert L.odtk_grad_to_atlas(1, 1, ctypes.cast(lv, ctypes.c_void_p), 36, ctypes.c_void_p(258), ctypes.c_void_p(256), 8, 16, 64,
                                None) == -1                                    # misaligned scale

    assert L.odtk_conv2d_dgrad(None, None) == -1
    e = engine.ConvDgradDesc()
    assert L.odtk_conv2d_dgrad(ctypes.byref(e), None) == -1
    b = e.base
    b.x, b.w, b.y = 256, 512, 1024
    b.n, b.h, b.width, b.cin, b.cout, b.ksize, b.out_mode = 1, 8, 16, 256, 256, 1, engine.OUT_NHWC_F16
    assert L.odtk_conv2d_dgrad(ctypes.byref(e), None) == -3                   # 3x3 only
    b.ksize, b.relu = 3, 1
    assert L.odtk_conv2d_dgrad(ctypes.byref(e), None) == -3                   # no ReLU on a gradient
    b.relu, b.out_mode = 0, engine.OUT_NCHW_F32
    assert L.odtk_conv2d_dgrad(ctypes.byref(e), None) == -3                   # NHWC fp16 only
    b.out_mode, b.stride = engine.OUT_NHWC_F16, 2
    assert L.odtk_conv2d_dgrad(ctypes.byref(e), None) == -3                   # stride 1 only
    b.stride = 1
    e.mask = 1026
    assert L.odtk_conv2d_dgrad(ctypes.byref(e), None) == -1                   # misaligned mask


@pytest.mark.parametrize("cout,cout_pad", [(256, 256), (36, 64), (54, 64), (720, 768)])
def test_pack_weight_dgrad_is_the_input_gradient(cout, cout_pad):
    """conv2d(g, repacked weights) == d/dx of the forward 3x3 convolution, in float64 (fp16-exact weights)."""
    g = torch.Generator().manual_seed(cout)
    cin = 128
    w = (torch.randn((cout, cin, 3, 3), generator=g) * 0.05).half().double()
    x = torch.randn((2, cin, 7, 11), generator=g, dtype=torch.float64, requires_grad=True)
    gy = torch.randn((2, cout, 7, 11), generator=g, dtype=torch.float64)
    ref, = torch.autograd.grad(F.conv2d(x, w, padding=1), x, gy)
    packed = engine.pack_weight_dgrad(w.float(), cout_pad)
    assert packed.shape == (cin, 9 * cout_pad) and packed.dtype == torch.float16
    wd = packed.double().view(cin, 3, 3, cout_pad).permute(0, 3, 1, 2)         # [cin, cout_pad, 3, 3]
    assert bool((wd[:, cout:] == 0).all())
    gpad = torch.cat([gy, gy.new_zeros((2, cout_pad - cout, 7, 11))], dim=1)
    out = F.conv2d(gpad, wd, padding=1)
    torch.testing.assert_close(out, ref, rtol=1e-12, atol=1e-12)
