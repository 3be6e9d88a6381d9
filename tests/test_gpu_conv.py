"""GPU parity tests of the tensor-core convolution engine (conv.cu / layers.cu) through the C ABI,
against torch's fp32 CPU convolution of the same fp16-rounded operands (the arithmetic the
reference's nn.Conv2d performs; torch is the oracle for this floating-point kernel).

Tolerance: operands are identical fp16 values on both sides, products are exact in fp32, so the only
differences are fp32 accumulation order and the final fp16 rounding of the output:
|err| <= 2e-3 * max|y| + 1e-3 for fp16 outputs, 1e-4 relative for fp32 outputs."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from retinanet_examples_b200 import engine

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _rand(shape, g, scale=1.0):
    return (torch.randn(shape, generator=g) * scale).to(torch.float16)


def _ref_conv(x_nhwc, w, bias, ksize, relu=False, residual=None, upsample=None, stride=1, pad=None):
    x = x_nhwc.float().permute(0, 3, 1, 2)
    y = F.conv2d(x, w.float(), bias.float() if bias is not None else None, stride=stride,
                 padding=ksize // 2 if pad is None else pad)
    if residual is not None:
        y = y + residual.float().permute(0, 3, 1, 2)
    if upsample is not None:
        y = y + F.interpolate(upsample.float().permute(0, 3, 1, 2), scale_factor=2)
    if relu:
        y = F.relu(y)
    return y   # NCHW fp32


def _close16(got_nhwc, ref_nchw):
    ref = ref_nchw.permute(0, 2, 3, 1)
    err = (got_nhwc.float().cpu() - ref).abs().max().item()
    tol = 2e-3 * ref.abs().max().item() + 1e-3
    assert err <= tol, (err, tol)


@pytest.mark.parametrize("n,h,w,cin,cout", [(1, 8, 16, 64, 64), (2, 13, 20, 256, 256), (1, 25, 40, 128, 512),
                                           (3, 7, 10, 512, 128), (1, 50, 80, 1024, 256), (2, 5, 5, 2048, 512)])
def test_conv1x1_matches_torch(n, h, w, cin, cout):
    g = torch.Generator().manual_seed(n * 1000 + cin + cout)
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, 1, 1), g, 0.05), torch.randn(cout, generator=g)
    y = engine.conv2d(x.to(DEV), engine.pack_weight(wt.float()).to(DEV), b.to(DEV), cout, 1, relu=True)
    _close16(y, _ref_conv(x, wt, b, 1, relu=True))


@pytest.mark.parametrize("n,h,w,cin,cout", [(1, 8, 16, 64, 64), (2, 13, 20, 256, 256), (1, 25, 40, 128, 128),
                                           (2, 7, 10, 256, 256), (1, 100, 160, 64, 64), (1, 50, 80, 512, 512),
                                           (2, 3, 3, 256, 256), (1, 33, 47, 128, 256)])
def test_conv3x3_matches_torch(n, h, w, cin, cout):
    g = torch.Generator().manual_seed(h * 100 + w + cin)
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, 3, 3), g, 0.03), torch.randn(cout, generator=g)
    y = engine.conv2d(x.to(DEV), engine.pack_weight(wt.float()).to(DEV), b.to(DEV), cout, 3)
    _close16(y, _ref_conv(x, wt, b, 3))


def test_conv_epilogue_residual_relu_and_upsample_add():
    g = torch.Generator().manual_seed(5)
    n, h, w, cin, cout = 2, 26, 40, 256, 256
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, 1, 1), g, 0.05), torch.randn(cout, generator=g)
    res, up = _rand((n, h, w, cout), g), _rand((n, h // 2, w // 2, cout), g)
    pw = engine.pack_weight(wt.float()).to(DEV)
    y = engine.conv2d(x.to(DEV), pw, b.to(DEV), cout, 1, relu=True, residual=res.to(DEV))
    _close16(y, _ref_conv(x, wt, b, 1, relu=True, residual=res))
    y = engine.conv2d(x.to(DEV), pw, b.to(DEV), cout, 1, upsample=up.to(DEV))
    _close16(y, _ref_conv(x, wt, b, 1, upsample=up))
    y = engine.conv2d(x.to(DEV), pw, None, cout, 1)
    _close16(y, _ref_conv(x, wt, None, 1))


@pytest.mark.parametrize("cout,mode", [(720, engine.OUT_NCHW_F32_SIGMOID), (36, engine.OUT_NCHW_F32),
                                       (162, engine.OUT_NCHW_F32), (720, engine.OUT_NCHW_F32)])
def test_head_final_conv_nchw_fp32(cout, mode):
    g = torch.Generator().manual_seed(cout)
    n, h, w, cin = 2, 25, 40, 256
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, 3, 3), g, 0.02), torch.randn(cout, generator=g)
    y = engine.conv2d(x.to(DEV), engine.pack_weight(wt.float()).to(DEV), b.to(DEV), cout, 3, out_mode=mode)
    ref = _ref_conv(x, wt, b, 3)
    if mode == engine.OUT_NCHW_F32_SIGMOID:
        ref = torch.sigmoid(ref)
    assert y.shape == ref.shape and y.dtype == torch.float32
    np.testing.assert_allclose(y.cpu().numpy(), ref.numpy(), rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("c,ks,stride,pad", [(64, 3, 2, 1), (128, 1, 2, 0), (256, 3, 2, 1), (3, 7, 2, 3)])
def test_lowered_strided_conv(c, ks, stride, pad):
    """stride-2 / 7x7 convolutions = receptive-field gather + GEMM rows."""
    g = torch.Generator().manual_seed(c * 10 + ks)
    n, h, w, cout = 2, 26, 38, 64
    x, wt, b = _rand((n, h, w, c), g), _rand((cout, c, ks, ks), g, 0.05), torch.randn(cout, generator=g)
    kreal = ks * ks * c
    kpad = (kreal + 63) // 64 * 64
    low = engine.lower_conv(x.to(DEV), ks, stride, pad, kpad=kpad if c % 8 else None)
    if c % 8 == 0:
        assert kreal % 64 == 0
    y = engine.conv2d(low, engine.pack_weight(wt.float(), kpad).to(DEV), b.to(DEV), cout, 1, relu=True)
    _close16(y, _ref_conv(x, wt, b, ks, relu=True, stride=stride, pad=pad))


def test_maxpool_matches_torch():
    g = torch.Generator().manual_seed(9)
    x = _rand((2, 21, 30, 64), g)
    y = engine.maxpool3x3s2(x.to(DEV))
    ref = F.max_pool2d(x.float().permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    np.testing.assert_array_equal(y.float().cpu().numpy(), ref.numpy())


@pytest.mark.parametrize("n,h,w", [(1, 32, 64), (2, 128, 256), (1, 226, 130)])
def test_stem_conv_overlapping_window_tma(n, h, w):
    """7x7 stride-2 stem through the zero-padded NHWC4 image + overlapping-window tensor map."""
    g = torch.Generator().manual_seed(h + w)
    x, wt, b = _rand((n, h, w, 3), g), _rand((64, 3, 7, 7), g, 0.1), torch.randn(64, generator=g)
    y = engine.stem_conv(x.to(DEV), engine.pack_stem_weight(wt.float()).to(DEV), b.to(DEV), 64, relu=True)
    _close16(y, _ref_conv(x, wt, b, 7, relu=True, stride=2, pad=3))


@pytest.mark.parametrize("n,h,w,cin,cout,ks", [(2, 26, 40, 64, 128, 3), (1, 50, 80, 256, 512, 1), (1, 100, 160, 128, 128, 3),
                                              (2, 8, 6, 512, 256, 3), (1, 200, 320, 256, 512, 1)])
def test_strided_conv_direct_tma(n, h, w, cin, cout, ks):
    """stride-2 1x1 / 3x3 convolutions through the parity-split 5-D tensor map (no gather)."""
    g = torch.Generator().manual_seed(h * 7 + cin)
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, ks, ks), g, 0.03), torch.randn(cout, generator=g)
    y = engine.conv2d(x.to(DEV), engine.pack_weight(wt.float()).to(DEV), b.to(DEV), cout, ks, relu=True, stride=2)
    _close16(y, _ref_conv(x, wt, b, ks, relu=True, stride=2, pad=ks // 2))


@pytest.mark.parametrize("ks,cin,cout,mode", [(1, 64, 256, 0), (3, 256, 256, 0), (1, 256, 64, 0), (3, 256, 720, 2), (1, 512, 2048, 0)])
def test_bias_added_on_the_tensor_core_equals_epilogue_bias(ks, cin, cout, mode):
    """bias_op (the packed hi/lo bias of odtk_conv_pack_bias) is accepted and does not change the result: the kernel adds
    the fp32 bias in its epilogue either way; both against torch."""
    g = torch.Generator().manual_seed(cout + ks)
    n, h, w = 2, 13, 20
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, ks, ks), g, 0.03), torch.randn(cout, generator=g) * 3
    pw, bd = engine.pack_weight(wt.float()).to(DEV), b.to(DEV)
    res = _rand((n, h, w, cout), g).to(DEV) if mode == 0 else None
    y0 = engine.conv2d(x.to(DEV), pw, bd, cout, ks, relu=(mode == 0), residual=res, out_mode=mode)
    y1 = engine.conv2d(x.to(DEV), pw, bd, cout, ks, relu=(mode == 0), residual=res, out_mode=mode, bias_op=engine.pack_bias(bd))
    assert torch.equal(y0, y1)
    if mode == 0:
        _close16(y1, _ref_conv(x, wt, b, ks, relu=True, residual=res.cpu()))
    else:
        ref = torch.sigmoid(_ref_conv(x, wt, b, ks)) if mode == engine.OUT_NCHW_F32_SIGMOID else _ref_conv(x, wt, b, ks)
        assert (y1.cpu() - ref).abs().max().item() <= 1e-4 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("n,h,w,cin,cout,ks", [(1, 100, 160, 256, 512, 3), (4, 100, 160, 256, 256, 3), (2, 200, 320, 64, 256, 1),
                                              (3, 100, 160, 128, 720, 3)])
def test_cluster_multicast_path(n, h, w, cin, cout, ks):
    """Large shapes with many 128-wide N tiles per M tile, incl. a ragged last M tile and the fp32 NCHW head
    epilogue over six N tiles (Cout 720)."""
    g = torch.Generator().manual_seed(n * 31 + cout)
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, ks, ks), g, 0.03), torch.randn(cout, generator=g)
    bd = b.to(DEV)
    if cout == 720:
        y = engine.conv2d(x.to(DEV), engine.pack_weight(wt.float()).to(DEV), bd, cout, ks, out_mode=engine.OUT_NCHW_F32,
                          bias_op=engine.pack_bias(bd))
        np.testing.assert_allclose(y.cpu().numpy(), _ref_conv(x, wt, b, ks).numpy(), rtol=2e-4, atol=2e-4)
    else:
        y = engine.conv2d(x.to(DEV), engine.pack_weight(wt.float()).to(DEV), bd, cout, ks, relu=True, bias_op=engine.pack_bias(bd))
        _close16(y, _ref_conv(x, wt, b, ks, relu=True))


# ---- 3x3 stride 1 (one shifted TMA box per tap and 64-channel chunk) --------------------------------------------------
# shapes chosen to hit: a single tile, ragged right/bottom edges, two channel chunks, several N tiles, 64 -> 64 layers
# with and without a residual, and the fp32 NCHW head outputs.
@pytest.mark.parametrize("n,h,w,cin,cout,bias_op,residual,relu", [
    (1, 16, 8, 64, 64, False, False, False), (1, 32, 24, 64, 64, True, False, True), (1, 40, 64, 64, 64, True, True, True),
    (2, 33, 47, 128, 128, False, False, True), (4, 48, 64, 256, 256, True, False, True), (1, 104, 160, 256, 256, True, False, False),
    (1, 9, 17, 64, 128, True, False, False), (2, 24, 16, 256, 512, True, False, True), (1, 8, 8, 128, 64, False, True, False)])
def test_conv3x3_halo_mode_matches_torch(n, h, w, cin, cout, bias_op, residual, relu):
    g = torch.Generator().manual_seed(h * 131 + w * 7 + cin + cout)
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, 3, 3), g, 0.03), torch.randn(cout, generator=g)
    res = _rand((n, h, w, cout), g) if residual else None
    bop = engine.pack_bias(b.to(DEV)) if bias_op else None
    y = engine.conv2d(x.to(DEV), engine.pack_weight(wt.float()).to(DEV), b.to(DEV), cout, 3, relu=relu,
                      residual=res.to(DEV) if residual else None, bias_op=bop)
    _close16(y, _ref_conv(x, wt, b, 3, relu=relu, residual=res))


@pytest.mark.parametrize("n,h,w,cout,mode", [(1, 48, 40, 36, engine.OUT_NCHW_F32), (2, 32, 40, 720, engine.OUT_NCHW_F32_SIGMOID),
                                            (1, 100, 160, 36, engine.OUT_NCHW_F32), (1, 25, 40, 720, engine.OUT_NCHW_F32)])
def test_conv3x3_halo_mode_head_outputs(n, h, w, cout, mode):
    g = torch.Generator().manual_seed(h + w + cout)
    x, wt, b = _rand((n, h, w, 256), g), _rand((cout, 256, 3, 3), g, 0.02), torch.randn(cout, generator=g)
    y = engine.conv2d(x.to(DEV), engine.pack_weight(wt.float()).to(DEV), b.to(DEV), cout, 3, out_mode=mode,
                      bias_op=engine.pack_bias(b.to(DEV)))
    ref = _ref_conv(x, wt, b, 3)
    if mode == engine.OUT_NCHW_F32_SIGMOID:
        ref = torch.sigmoid(ref)
    err = (y.cpu() - ref).abs().max().item()
    assert err <= 1e-4 * max(1.0, ref.abs().max().item()), err


@pytest.mark.parametrize("n,h,w", [(1, 32, 16), (2, 34, 50), (1, 800, 1280)])
def test_stem_raw_window_mode_edges(n, h, w):
    """7x7 stem on sizes whose output patches are ragged, and on the benchmark's full size."""
    g = torch.Generator().manual_seed(h * 3 + w)
    x, wt, b = _rand((n, h, w, 3), g), _rand((64, 3, 7, 7), g, 0.1), torch.randn(64, generator=g)
    y = engine.stem_conv(x.to(DEV), engine.pack_stem_weight(wt.float()).to(DEV), b.to(DEV), 64, relu=True)
    _close16(y, _ref_conv(x, wt, b, 7, relu=True, stride=2, pad=3))


# ---- kernel-variant assertions (odtk_conv_last_plan), epilogue upsample-add, element-strided stride 2 ---------------
@pytest.mark.parametrize("n,h,w,cin,cout", [(2, 26, 48, 256, 256), (1, 100, 160, 512, 256), (3, 10, 16, 1024, 256),
                                           (1, 50, 80, 128, 512)])
def test_upsample_add_on_the_tensor_core(n, h, w, cin, cout):
    """FPN lateral 1x1 + nearest-upsample add in the fp32 epilogue of the GEMM-row kernel."""
    g = torch.Generator().manual_seed(h * 17 + w + cin)
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, 1, 1), g, 0.05), torch.randn(cout, generator=g)
    up = _rand((n, h // 2, w // 2, cout), g)
    bd = b.to(DEV)
    y = engine.conv2d(x.to(DEV), engine.pack_weight(wt.float()).to(DEV), bd, cout, 1, upsample=up.to(DEV),
                      bias_op=engine.pack_bias(bd))
    plan = engine.last_plan()
    assert plan["up_mma"] == 0 and plan["mode"] == 0, plan
    _close16(y, _ref_conv(x, wt, b, 1, upsample=up))


def test_upsample_add_epilogue_fallback_when_rows_do_not_split():
    g = torch.Generator().manual_seed(77)
    n, h, w, cin, cout = 1, 26, 40, 256, 256           # W % 16 != 0
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, 1, 1), g, 0.05), torch.randn(cout, generator=g)
    up = _rand((n, h // 2, w // 2, cout), g)
    y = engine.conv2d(x.to(DEV), engine.pack_weight(wt.float()).to(DEV), b.to(DEV), cout, 1, upsample=up.to(DEV))
    assert engine.last_plan()["up_mma"] == 0
    _close16(y, _ref_conv(x, wt, b, 1, upsample=up))


@pytest.mark.parametrize("n,h,w,cin,cout,ks", [(2, 25, 40, 2048, 256, 3), (2, 13, 20, 256, 256, 3), (1, 25, 39, 128, 128, 3),
                                              (3, 7, 9, 512, 256, 1), (1, 51, 81, 64, 64, 3), (32, 25, 40, 512, 256, 3)])
def test_strided_conv_odd_sizes_element_strided_tma(n, h, w, cin, cout, ks):
    """stride-2 convolutions on ODD sizes (FPN pyramid6 / pyramid7 at 25x40 / 13x20): element-strided TMA boxes,
    no receptive-field gather."""
    g = torch.Generator().manual_seed(h * 7 + w + cin + ks)
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, ks, ks), g, 0.02), torch.randn(cout, generator=g)
    bd = b.to(DEV)
    y = engine.conv2d(x.to(DEV), engine.pack_weight(wt.float()).to(DEV), bd, cout, ks, relu=True, stride=2,
                      bias_op=engine.pack_bias(bd))
    plan = engine.last_plan()
    assert plan["mode"] == 1, plan
    assert tuple(y.shape) == (n, (h - 1) // 2 + 1, (w - 1) // 2 + 1, cout)
    _close16(y, _ref_conv(x, wt, b, ks, relu=True, stride=2, pad=ks // 2))


def test_relu_copy():
    g = torch.Generator().manual_seed(3)
    x = _rand((2, 13, 20, 256), g)
    y = engine.relu(x.to(DEV))
    np.testing.assert_array_equal(y.float().cpu().numpy(), F.relu(x.float()).numpy())


@pytest.mark.parametrize("shape,ks,kw,expect", [
    ((4, 100, 160, 256, 256), 3, {}, {"mode": 1, "bn": 128, "num_n_tiles": 2}),             # shifted box per tap, 128-wide N tiles
    ((2, 200, 320, 64, 64), 3, {}, {"mode": 1, "bn": 64}),
    ((2, 50, 80, 256, 1024), 1, {"residual": True}, {"mode": 0, "bn": 128, "num_n_tiles": 8}),   # residual in the epilogue
    ((8, 50, 80, 1024, 256), 1, {}, {"mode": 0, "bn": 128, "nstages": 6}),
    ((4, 25, 40, 512, 2048), 1, {"residual": True}, {"mode": 0, "bn": 128}),
    ((19, 25, 40, 2048, 512), 1, {}, {"mode": 0, "num_m_tiles": 149}),                      # ragged last M tile
    ((11, 100, 160, 512, 256), 1, {}, {"mode": 0, "bn": 128, "grid": 132}),                 # persistent: one CTA per SM
    ((2, 200, 320, 256, 64), 1, {}, {"mode": 0, "bn": 64}),
    ((2, 100, 160, 512, 1024), 1, {"stride": 2}, {"mode": 3}),                             # even stride 2: parity split
    ((32, 7, 10, 256, 256), 3, {}, {"mode": 1, "bn": 64}),                                 # few tiles: narrower N tile
    ((2, 100, 160, 128, 512), 1, {"residual": True}, {"mode": 0, "bn": 128}),
    ((2, 100, 160, 256, 36), 3, {"f32": True}, {"mode": 1, "bn": 64, "num_n_tiles": 1}),      # narrow head output
])
def test_conv_variant_selection(shape, ks, kw, expect):
    """The host code picks the kernel variant from the shape; assert which one ran AND that it is right."""
    n, h, w, cin, cout = shape
    g = torch.Generator().manual_seed(sum(shape) + ks)
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, ks, ks), g, 0.03), torch.randn(cout, generator=g)
    stride = kw.get("stride", 1)
    res = _rand((n, h, w, cout), g) if kw.get("residual") else None
    bd = b.to(DEV)
    f32 = kw.get("f32", False)
    y = engine.conv2d(x.to(DEV), engine.pack_weight(wt.float()).to(DEV), bd, cout, ks, relu=not f32,
                      residual=res.to(DEV) if res is not None else None, stride=stride, bias_op=engine.pack_bias(bd),
                      out_mode=engine.OUT_NCHW_F32 if f32 else engine.OUT_NHWC_F16)
    plan = engine.last_plan()
    for k, v in expect.items():
        assert plan[k] == v, (k, plan)
    if f32:
        ref = _ref_conv(x, wt, b, ks)
        assert (y.cpu() - ref).abs().max().item() <= 1e-4 * max(1.0, ref.abs().max().item())
    else:
        _close16(y, _ref_conv(x, wt, b, ks, relu=True, residual=res, stride=stride, pad=ks // 2))


def test_tensor_map_cache_hits_on_repeated_calls():
    import ctypes
    from retinanet_examples_b200 import _lib
    g = torch.Generator().manual_seed(11)
    x, wt = _rand((1, 16, 16, 64), g).to(DEV), engine.pack_weight(_rand((64, 64, 3, 3), g, 0.05).float()).to(DEV)
    out = torch.empty((1, 16, 16, 64), dtype=torch.float16, device=DEV)
    h0, m0, h1, m1 = (ctypes.c_longlong(0) for _ in range(4))
    engine.conv2d(x, wt, None, 64, 3, out=out)
    _lib.lib().odtk_conv_map_cache_stats(ctypes.byref(h0), ctypes.byref(m0))
    engine.conv2d(x, wt, None, 64, 3, out=out)
    _lib.lib().odtk_conv_map_cache_stats(ctypes.byref(h1), ctypes.byref(m1))
    assert m1.value == m0.value and h1.value > h0.value


@pytest.mark.parametrize("n,h,w", [(1, 32, 16), (2, 34, 50), (1, 226, 130), (2, 128, 256), (1, 800, 1280), (3, 28, 28)])
def test_stem_pool_fused_equals_stem_then_maxpool(n, h, w):
    """conv1 + bn1 + relu + maxpool in one call (odtk_stem_pool): bit-identical to the two-kernel route (the same fp16
    values are pooled), and within the fp16 bar of torch's fp32 conv + max_pool2d."""
    g = torch.Generator().manual_seed(h * 5 + w)
    x, wt, b = _rand((n, h, w, 3), g), _rand((64, 3, 7, 7), g, 0.1), torch.randn(64, generator=g)
    ws, bd = engine.pack_stem_weight(wt.float()).to(DEV), b.to(DEV)
    fused = engine.stem_pool(x.to(DEV), ws, bd, 64, relu=True)
    two = engine.maxpool3x3s2(engine.stem_conv(x.to(DEV), ws, bd, 64, relu=True))
    assert fused.shape == two.shape
    np.testing.assert_array_equal(fused.float().cpu().numpy(), two.float().cpu().numpy())
    ref = F.max_pool2d(_ref_conv(x, wt, b, 7, relu=True, stride=2, pad=3), 3, 2, 1)
    _close16(fused, ref)


def test_pad_input_rows_kernel_matches_per_pixel_layout():
    """odtk_pad_input, W % 8 == 0 (row-staged kernel) and W % 8 != 0 (per-pixel kernel): NHWC3 -> zero-bordered NHWC4."""
    import ctypes
    from retinanet_examples_b200 import _lib
    g = torch.Generator().manual_seed(4)
    for (n, h, w) in ((2, 10, 16), (1, 7, 13), (1, 64, 1280)):
        x = _rand((n, h, w, 3), g).to(DEV)
        xp = torch.full((n, h + 6, w + 8, 4), 7.0, dtype=torch.float16, device=DEV)
        _lib.check(_lib.lib().odtk_pad_input(ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(xp.data_ptr()), n, h, w,
                                             ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "pad_input")
        ref = torch.zeros((n, h + 6, w + 8, 4), dtype=torch.float16, device=DEV)
        ref[:, 3:3 + h, 3:3 + w, :3] = x
        np.testing.assert_array_equal(xp.float().cpu().numpy(), ref.float().cpu().numpy())


@pytest.mark.parametrize("n,h,w,c,groups,stride", [(2, 24, 32, 128, 32, 1), (1, 50, 80, 256, 32, 1), (2, 26, 40, 512, 32, 2),
                                                  (1, 25, 39, 256, 32, 2), (1, 16, 16, 1024, 32, 1), (2, 20, 24, 256, 32 // 2, 1)])
def test_grouped_conv3x3_resnext(n, h, w, c, groups, stride):
    """Grouped 3x3 (ResNeXt conv2, torchvision groups=32): each 64-channel output block reads only its own input chunk
    (block-diagonal weights), stride 1, even stride 2 (parity split) and odd stride 2 (element-strided boxes)."""
    g = torch.Generator().manual_seed(c + groups + h)
    x, wt, b = _rand((n, h, w, c), g), _rand((c, c // groups, 3, 3), g, 0.1), torch.randn(c, generator=g)
    bd = b.to(DEV)
    y = engine.conv2d(x.to(DEV), engine.pack_weight_grouped(wt.float(), groups).to(DEV), bd, c, 3, relu=True, stride=stride,
                      bias_op=engine.pack_bias(bd), groups=groups)
    plan = engine.last_plan()
    assert plan["bn"] == 64 and plan["num_n_tiles"] == c // 64, plan
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), b, stride=stride, padding=1, groups=groups)
    _close16(y, F.relu(ref))


@pytest.mark.parametrize("n,h,w,c1", [(2, 24, 48, 64), (1, 9, 17, 64), (3, 8, 16, 128), (1, 20, 40, 128), (2, 13, 21, 64),
                                      (4, 200, 320, 64), (2, 100, 160, 128)])
def test_bottleneck_tail_fused_matches_torch_and_two_kernel_route(n, h, w, c1):
    """conv2 (3x3) + bn + relu + conv3 (1x1) + bn + identity + relu in one call (odtk_bottleneck_tail): against torch fp32 with
    the intermediate rounded to fp16 (what the two-kernel route stores), and against the two-kernel route itself
    (conv.cu 3x3, then 1x1 + residual).  Ragged tiles, an odd tile count and
    many tiles per CTA are covered."""
    c2 = 4 * c1
    g = torch.Generator().manual_seed(n * 7 + h + w + c1)
    x = _rand((n, h, w, c1), g)
    w2, b2 = _rand((c1, c1, 3, 3), g, 0.04), torch.randn(c1, generator=g) * 0.5
    w3, b3 = _rand((c2, c1, 1, 1), g, 0.08), torch.randn(c2, generator=g) * 0.5
    res = _rand((n, h, w, c2), g)
    w2p, w3p = engine.pack_weight(w2.float()).to(DEV), engine.pack_weight(w3.float()).to(DEV)
    xd, rd, b2d, b3d = x.to(DEV), res.to(DEV), b2.to(DEV), b3.to(DEV)
    y = engine.bottleneck_tail(xd, w2p, b2d, w3p, b3d, rd, relu=True)
    torch.cuda.synchronize()
    mid = _ref_conv(x, w2, b2, 3, relu=True).permute(0, 2, 3, 1).to(torch.float16)          # fp16, as stored between the kernels
    _close16(y, _ref_conv(mid, w3, b3, 1, relu=True, residual=res))
    mid_d = engine.conv2d(xd, w2p, b2d, c1, 3, relu=True, bias_op=engine.pack_bias(b2d))
    y2 = engine.conv2d(mid_d, w3p, b3d, c2, 1, relu=True, residual=rd, bias_op=engine.pack_bias(b3d))
    err = (y.float() - y2.float()).abs().max().item()
    assert err <= 2e-3 * y2.float().abs().max().item() + 1e-3, err


@pytest.mark.parametrize("n,h,w", [(2, 24, 48), (1, 9, 17), (3, 8, 16), (2, 200, 320)])
def test_bottleneck_tail_with_projected_identity(n, h, w):
    """First block of layer1: the identity is a 1x1 projection (torchvision `downsample`) of the 64-channel block input,
    computed by the fused kernel on the tensor core instead of being read from HBM."""
    c1, c2 = 64, 256
    g = torch.Generator().manual_seed(n * 11 + h + w)
    xin = _rand((n, h, w, 64), g)
    x = _rand((n, h, w, c1), g)
    w2, b2 = _rand((c1, c1, 3, 3), g, 0.04), torch.randn(c1, generator=g) * 0.5
    w3, b3 = _rand((c2, c1, 1, 1), g, 0.08), torch.randn(c2, generator=g) * 0.5
    wd, bd = _rand((c2, 64, 1, 1), g, 0.1), torch.randn(c2, generator=g) * 0.5
    y = engine.bottleneck_tail(x.to(DEV), engine.pack_weight(w2.float()).to(DEV), b2.to(DEV), engine.pack_weight(w3.float()).to(DEV),
                               (b3 + bd).to(DEV), None, relu=True, xproj=xin.to(DEV), wproj=engine.pack_weight(wd.float()).to(DEV))
    torch.cuda.synchronize()
    mid = _ref_conv(x, w2, b2, 3, relu=True).permute(0, 2, 3, 1).to(torch.float16)
    ref = F.relu(_ref_conv(mid, w3, b3, 1) + _ref_conv(xin, wd, bd, 1))
    _close16(y, ref)


@pytest.mark.parametrize("n,h,w,c,stride", [(2, 16, 24, 64, 1), (1, 25, 39, 192, 2), (3, 7, 10, 384, 1), (1, 100, 160, 192, 2)])
def test_depthwise3x3_relu6_matches_torch(n, h, w, c, stride):
    """Depthwise 3x3 + bias + ReLU6 (MobileNetV2's inverted residual blocks): fp16 operands, fp32 accumulation."""
    g = torch.Generator().manual_seed(h * 7 + w + c)
    x, wt, b = _rand((n, h, w, c), g, 2.0), _rand((c, 1, 3, 3), g, 0.5), torch.randn(c, generator=g)
    wp = wt.float().reshape(c, 9).t().contiguous().to(torch.float16)
    y = engine.depthwise3x3(x.to(DEV), wp.to(DEV), b.to(DEV), stride=stride, act=2)
    ref = F.relu6(F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), b, stride=stride, padding=1, groups=c))
    _close16(y, ref)


def test_conv1x1_relu6_epilogue():
    g = torch.Generator().manual_seed(77)
    x, wt, b = _rand((2, 13, 20, 128), g, 2.0), _rand((192, 128, 1, 1), g, 0.2), torch.randn(192, generator=g) * 3
    bd = b.to(DEV)
    y = engine.conv2d(x.to(DEV), engine.pack_weight(wt.float()).to(DEV), bd, 192, 1, relu=2, bias_op=engine.pack_bias(bd))
    ref = F.relu6(_ref_conv(x, wt, b, 1))
    assert float(ref.max()) == 6.0 and float(ref.min()) == 0.0       # both clamps are exercised
    _close16(y, ref)


def test_conv1x1_n_tile_not_a_multiple_of_64():
    """Cout = 960 (MobileNetV2's widest expansion) on enough pixels for 128-wide N tiles: the eighth tile is half outside
    Cout, its weight rows are zero-filled by the TMA unit and its columns must not be stored."""
    g = torch.Generator().manual_seed(960)
    x, wt, b = _rand((1, 48, 48, 192), g), _rand((960, 192, 1, 1), g, 0.1), torch.randn(960, generator=g)
    bd = b.to(DEV)
    y = engine.conv2d(x.to(DEV), engine.pack_weight(wt.float()).to(DEV), bd, 960, 1, relu=2, bias_op=engine.pack_bias(bd))
    assert engine.last_plan()["bn"] == 128 and engine.last_plan()["num_n_tiles"] == 8
    _close16(y, F.relu6(_ref_conv(x, wt, b, 1)))


@pytest.mark.parametrize("n,h,w,c3", [(2, 24, 48, 64), (1, 9, 17, 64), (3, 8, 16, 128), (2, 200, 320, 64), (2, 200, 320, 128)])
def test_bottleneck_tail_with_next_conv1(n, h, w, c3):
    """GEMM3 of the fused tail kernel: the NEXT block's conv1 (1x1 + bias + ReLU) computed from the block output while its
    chunks are still in shared memory; the block output itself must be unchanged."""
    c1, c2 = 64, 256
    g = torch.Generator().manual_seed(n * 13 + h + w + c3)
    x = _rand((n, h, w, c1), g)
    w2, b2 = _rand((c1, c1, 3, 3), g, 0.04), torch.randn(c1, generator=g) * 0.5
    w3, b3 = _rand((c2, c1, 1, 1), g, 0.08), torch.randn(c2, generator=g) * 0.5
    w1n, b1n = _rand((c3, c2, 1, 1), g, 0.06), torch.randn(c3, generator=g) * 0.5
    res = _rand((n, h, w, c2), g)
    args = (x.to(DEV), engine.pack_weight(w2.float()).to(DEV), b2.to(DEV), engine.pack_weight(w3.float()).to(DEV), b3.to(DEV), res.to(DEV))
    y0 = engine.bottleneck_tail(*args, relu=True)
    y, z = engine.bottleneck_tail(*args, relu=True, w_next=engine.pack_weight(w1n.float()).to(DEV), b_next=b1n.to(DEV))
    torch.cuda.synchronize()
    assert torch.equal(y, y0)
    _close16(z, _ref_conv(y0.cpu(), w1n, b1n, 1, relu=True))
