"""CPU tests of the full-precision mode's host side: the split-TF32 weight packing, the new C-ABI entry points and
Model.set_precision("fp32")'s argument checks."""
import ctypes

import pytest
import torch

from retinanet_examples_b200 import _lib, engine
from retinanet_examples_b200.model import FP32_BACKBONES, Model


def _bits(t):
    return t.contiguous().view(torch.int32)


def test_split_packing_is_tf32_valued_and_exact_to_2e22():
    g = torch.Generator().manual_seed(0)
    w = torch.randn((64, 32, 3, 3), generator=g) * torch.logspace(-6, 3, 64).view(-1, 1, 1, 1)
    hi, lo = engine.pack_weight_tf32x2(w)
    assert hi.shape == lo.shape == (64, 9 * 32) and hi.dtype == lo.dtype == torch.float32
    assert int((_bits(hi) & 0x1FFF).count_nonzero()) == 0
    assert int((_bits(lo) & 0x1FFF).count_nonzero()) == 0
    ref = w.permute(0, 2, 3, 1).reshape(64, -1).double()
    err = (ref - hi.double() - lo.double()).abs()
    assert bool((err <= 2.0 ** -22 * ref.abs()).all()), float((err / ref.abs()).max())
    # hi is the nearest tf32 value: |w - hi| <= half a tf32 ulp (2^-11 relative)
    assert bool(((ref - hi.double()).abs() <= 2.0 ** -11 * ref.abs()).all())


def test_split_packing_pads_k():
    hi, lo = engine.pack_weight_tf32x2(torch.ones((4, 3, 1, 1)), kpad=32)
    assert hi.shape == (4, 32) and bool((hi[:, 3:] == 0).all()) and bool((lo == 0).all())


def test_rna_ties_round_away_from_zero():
    one = 1.0
    ulp = 2.0 ** -10                                                   # tf32 spacing in [1, 2)
    x = torch.tensor([one + ulp / 2, -(one + ulp / 2), one + 3 * ulp / 2, one + ulp / 2 - 2.0 ** -23, 0.0, -0.0])
    r = engine.tf32_rna(x)
    assert r.tolist()[:4] == [one + ulp, -(one + ulp), one + 2 * ulp, one]
    assert _bits(r[4:]).tolist() == _bits(x[4:]).tolist()


def test_stem_packing_k_order():
    w = torch.randn((16, 3, 7, 7), generator=torch.Generator().manual_seed(1))
    hi, lo = engine.pack_stem_weight_tf32x2(w)
    assert hi.shape == (16, 224)
    k = hi.view(16, 7, 8, 4)
    assert bool((k[:, :, 7] == 0).all()) and bool((k[:, :, :, 3] == 0).all())
    assert torch.equal(k[:, :, :7, :3], engine.tf32_rna(w.permute(0, 2, 3, 1)))
    assert torch.allclose((hi + lo).view(16, 7, 8, 4)[:, :, :7, :3], w.permute(0, 2, 3, 1), rtol=2.0 ** -22, atol=0)


def test_new_signatures_resolve():
    L = _lib.lib()
    for name in ("odtk_conv2d_f32", "odtk_pad_input_f32", "odtk_preprocess_u8_f32", "odtk_preprocess_resize_u8_f32",
                 "odtk_maxpool3x3s2_f32", "odtk_relu_copy_rows_f32"):
        assert name in _lib.SIGNATURES
        assert getattr(L, name).argtypes == _lib.SIGNATURES[name][1]


def test_conv_f32_rejects_bad_descriptors_without_a_gpu():
    """Argument checks run before any CUDA call: a null descriptor / pointers are ODTK_E_INVALID."""
    L = _lib.lib()
    assert L.odtk_conv2d_f32(None, None) == -1
    d = engine.ConvF32Desc()
    assert L.odtk_conv2d_f32(ctypes.byref(d), None) == -1


def test_set_precision_argument_checks():
    assert set(FP32_BACKBONES) == {"ResNet18FPN", "ResNet34FPN", "ResNet50FPN", "ResNet101FPN", "ResNet152FPN"}
    for bb in ("ResNeXt50_32x4dFPN", "ResNeXt101_32x8dFPN", "MobileNetV2FPN"):
        with pytest.raises(ValueError, match="full precision"):
            Model(bb, classes=3).set_precision("fp32")
    m = Model("ResNet18FPN", classes=3)
    with pytest.raises(ValueError, match="precision must be"):
        m.set_precision("fp64")
    with pytest.raises(ValueError, match="precision must be"):
        m.set_precision("tf32")
    assert m.set_precision("fp32").precision == "fp32"
    assert m.set_precision("fp16").precision == "fp16"
