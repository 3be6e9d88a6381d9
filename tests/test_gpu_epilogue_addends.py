"""GPU tests of the fp16 epilogues' addend and bias loads: conv_gemm_kernel folds the bias into the accumulators before
any store and loads the residual / upsample / mask addends of 64 columns at a time ahead of that chunk's stores, and the
bottleneck tail loads each output tile's residual before the tile's MMAs.  The cases cover the edges of that staging:
ragged last M tiles (mode 0), patches clipped at odd image borders, Cout that ends inside a 64-column chunk, each N tile
(64 / 128 / 256, chosen through the launch budget as in test_gpu_conv_wide.py), NCHW outputs, the masked input gradient
with its residual, and the tail at odd sizes with and without the projected identity and the next block's conv1.  Each
is checked against a CUDA fp32 torch convolution (TF32 off) within the fp16 bound of test_gpu_conv.py, and, where the
same result has another route through the library, for identical bits."""
import pytest
import torch
import torch.nn.functional as F

from retinanet_examples_b200 import _lib, engine

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _fp32_reference():
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = old


def _rand(shape, g, scale=1.0):
    return (torch.randn(shape, generator=g) * scale).to(torch.float16).to(DEV)


def _close16(got_nhwc, ref_nchw):
    ref = ref_nchw.permute(0, 2, 3, 1)
    err = (got_nhwc.float() - ref).abs().max().item()
    tol = 2e-3 * ref.abs().max().item() + 1e-3
    assert err <= tol, (err, tol)


def _ref_conv(x_nhwc, w, bias, ksize, relu=0, residual=None, upsample=None):
    y = F.conv2d(x_nhwc.float().permute(0, 3, 1, 2), w.float(), bias, padding=ksize // 2)
    if residual is not None:
        y = y + residual.float().permute(0, 3, 1, 2)
    if upsample is not None:
        y = y + F.interpolate(upsample.float().permute(0, 3, 1, 2), scale_factor=2)
    if relu:
        y = F.relu6(y) if relu == 2 else F.relu(y)
    return y


def _with_budget(sms, fn):
    _lib.lib().odtk_set_sm_budget(sms)
    try:
        out = fn()
        plan = engine.last_plan()
        torch.cuda.synchronize()
    finally:
        _lib.lib().odtk_set_sm_budget(0)
    return out, plan


def _every_tile_width(fn, cout):
    """fn() on each N tile the launch budget can select for this shape: {bn: result}."""
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    y, plan = _with_budget(2, fn)
    outs = {plan["bn"]: y}
    n128 = plan["num_m_tiles"] * ((cout + 127) // 128)
    for budget in (min(n128, sms) & ~1, n128 + 1):
        if 2 <= budget <= sms:
            y, plan = _with_budget(budget, fn)
            outs.setdefault(plan["bn"], y)
    return outs


# (n, h, w, cin, cout, ksize): M = n*h*w not a multiple of 128; 3x3 patches clipped at odd borders; Cout 720 and 192 end
# inside a 64-column chunk of the last N tile
CASES = [(2, 27, 29, 256, 512, 1), (2, 19, 27, 128, 720, 1), (1, 61, 53, 256, 192, 1), (2, 29, 43, 256, 512, 3),
         (1, 27, 45, 128, 720, 3), (4, 21, 37, 64, 256, 3)]


@pytest.mark.parametrize("n,h,w,cin,cout,ks", CASES)
def test_residual_and_bias_on_every_tile_width(n, h, w, cin, cout, ks):
    g = torch.Generator().manual_seed(n * 5 + h * 3 + w + cin + cout + ks)
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, ks, ks), g, 0.03), torch.randn(cout, generator=g).to(DEV)
    res = _rand((n, h, w, cout), g)
    pw = engine.pack_weight(wt.float())
    outs = _every_tile_width(lambda: engine.conv2d(x, pw, b, cout, ks, relu=True, residual=res), cout)
    assert {128, 256} <= set(outs), sorted(outs)
    ref = _ref_conv(x, wt, b, ks, relu=True, residual=res)
    first = next(iter(outs.values()))
    for bn, y in outs.items():
        _close16(y, ref)
        assert torch.equal(y, first), bn
    # no bias: the residual alone, including the -0.0 of acc + residual
    outs = _every_tile_width(lambda: engine.conv2d(x, pw, None, cout, ks, residual=res), cout)
    ref = _ref_conv(x, wt, None, ks, residual=res)
    for y in outs.values():
        _close16(y, ref)


@pytest.mark.parametrize("n,h,w,cin,cout", [(2, 40, 48, 256, 256), (1, 42, 46, 128, 512), (2, 38, 40, 256, 256)])
def test_residual_and_upsample_together(n, h, w, cin, cout):
    """Both addends in one epilogue (the fp16 sum order is acc + bias, + residual, + upsample), on every tile width; W % 16
    != 0 in the last case (the epilogue upsample path)."""
    g = torch.Generator().manual_seed(h * 13 + w + cin + cout)
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, 1, 1), g, 0.05), torch.randn(cout, generator=g).to(DEV)
    res, up = _rand((n, h, w, cout), g), _rand((n, h // 2, w // 2, cout), g)
    pw = engine.pack_weight(wt.float())
    outs = _every_tile_width(lambda: engine.conv2d(x, pw, b, cout, 1, residual=res, upsample=up), cout)
    assert {128, 256} <= set(outs), sorted(outs)
    ref = _ref_conv(x, wt, b, 1, residual=res, upsample=up)
    first = next(iter(outs.values()))
    for bn, y in outs.items():
        _close16(y, ref)
        assert torch.equal(y, first), bn


@pytest.mark.parametrize("cout,mode", [(36, engine.OUT_NCHW_F32), (720, engine.OUT_NCHW_F32_SIGMOID),
                                       (512, engine.OUT_NCHW_F32_SIGMOID)])
def test_nchw_outputs_with_the_folded_bias(cout, mode):
    g = torch.Generator().manual_seed(cout * 3 + mode)
    n, h, w, cin = 2, 13, 19, 256
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, 3, 3), g, 0.02), torch.randn(cout, generator=g).to(DEV)
    pw = engine.pack_weight(wt.float())
    outs = _every_tile_width(lambda: engine.conv2d(x, pw, b, cout, 3, out_mode=mode), cout)
    ref = _ref_conv(x, wt, b, 3)
    if mode == engine.OUT_NCHW_F32_SIGMOID:
        ref = torch.sigmoid(ref)
    first = next(iter(outs.values()))
    for bn, y in outs.items():
        assert torch.equal(y, first), bn
        err = (y - ref).abs().max().item()
        assert err <= 2e-3 * ref.abs().max().item() + 1e-3, err


@pytest.mark.parametrize("n,h,w,cout", [(2, 13, 21, 256), (1, 9, 33, 128)])
def test_masked_dgrad_with_residual(n, h, w, cout):
    """The masked input-gradient instance: + residual, then zero where the saved input is not > 0."""
    g = torch.Generator().manual_seed(n + h * 7 + w + cout)
    cpad = 64
    gr = _rand((n, h, w, cpad), g, 0.3)
    wt = (torch.randn((cpad, cout, 3, 3), generator=g) * 0.05).half().float().to(DEV)   # forward: cout -> cpad
    res, mask = _rand((n, h, w, cout), g), _rand((n, h, w, cout), g)
    got = engine.conv2d_dgrad(gr, engine.pack_weight_dgrad(wt, cpad), cout, mask=mask, residual=res)
    xx = torch.zeros((n, cout, h, w), device=DEV, requires_grad=True)
    gx, = torch.autograd.grad(F.conv2d(xx, wt, padding=1), xx, gr.float().permute(0, 3, 1, 2))
    ref = torch.where(mask.float().permute(0, 3, 1, 2) > 0, gx + res.float().permute(0, 3, 1, 2), torch.zeros_like(gx))
    _close16(got, ref)


def _tail_operands(n, h, w, c1, c2, g):
    x = _rand((n, h, w, c1), g)
    w2, b2 = _rand((c1, c1, 3, 3), g, 0.04), torch.randn(c1, generator=g).to(DEV) * 0.5
    w3, b3 = _rand((c2, c1, 1, 1), g, 0.08), torch.randn(c2, generator=g).to(DEV) * 0.5
    return x, w2, b2, w3, b3


@pytest.mark.parametrize("n,h,w,c1,relu", [(1, 11, 19, 64, True), (2, 7, 13, 128, True), (1, 23, 29, 128, False),
                                           (3, 5, 37, 64, False)])
def test_tail_residual_at_odd_sizes(n, h, w, c1, relu):
    """Identity from HBM, loaded before the output tile's MMAs: against torch and bit for bit against the two-kernel
    route (3x3, then 1x1 + residual)."""
    c2 = 4 * c1
    g = torch.Generator().manual_seed(n * 3 + h * 5 + w + c1)
    x, w2, b2, w3, b3 = _tail_operands(n, h, w, c1, c2, g)
    res = _rand((n, h, w, c2), g)
    w2p, w3p = engine.pack_weight(w2.float()), engine.pack_weight(w3.float())
    y = engine.bottleneck_tail(x, w2p, b2, w3p, b3, res, relu=relu)
    mid = engine.conv2d(x, w2p, b2, c1, 3, relu=True)
    y2 = engine.conv2d(mid, w3p, b3, c2, 1, relu=relu, residual=res)
    torch.cuda.synchronize()
    assert torch.equal(y, y2)
    ref_mid = _ref_conv(x, w2, b2, 3, relu=True).permute(0, 2, 3, 1).to(torch.float16)
    _close16(y, _ref_conv(ref_mid, w3, b3, 1, relu=relu, residual=res))


@pytest.mark.parametrize("n,h,w", [(1, 11, 19), (2, 9, 27)])
def test_tail_projection_at_odd_sizes(n, h, w):
    c1, c2 = 64, 256
    g = torch.Generator().manual_seed(n * 17 + h + w)
    x, w2, b2, w3, b3 = _tail_operands(n, h, w, c1, c2, g)
    xin = _rand((n, h, w, 64), g)
    wd, bd = _rand((c2, 64, 1, 1), g, 0.1), torch.randn(c2, generator=g).to(DEV) * 0.5
    y = engine.bottleneck_tail(x, engine.pack_weight(w2.float()), b2, engine.pack_weight(w3.float()), b3 + bd, None,
                               relu=True, xproj=xin, wproj=engine.pack_weight(wd.float()))
    torch.cuda.synchronize()
    mid = _ref_conv(x, w2, b2, 3, relu=True).permute(0, 2, 3, 1).to(torch.float16)
    _close16(y, F.relu(_ref_conv(mid, w3, b3, 1) + _ref_conv(xin, wd, bd, 1)))


@pytest.mark.parametrize("n,h,w,c3", [(1, 11, 19, 64), (2, 7, 13, 128), (1, 17, 9, 128)])
def test_tail_next_conv1_at_odd_sizes(n, h, w, c3):
    """GEMM3 (the instance whose consumers now take 232 registers): y unchanged by it, z bit for bit the separate 1x1."""
    c1, c2 = 64, 256
    g = torch.Generator().manual_seed(n * 19 + h + w + c3)
    x, w2, b2, w3, b3 = _tail_operands(n, h, w, c1, c2, g)
    res = _rand((n, h, w, c2), g)
    w1n, b1n = _rand((c3, c2, 1, 1), g, 0.06), torch.randn(c3, generator=g).to(DEV) * 0.5
    args = (x, engine.pack_weight(w2.float()), b2, engine.pack_weight(w3.float()), b3, res)
    y0 = engine.bottleneck_tail(*args, relu=True)
    y, z = engine.bottleneck_tail(*args, relu=True, w_next=engine.pack_weight(w1n.float()), b_next=b1n)
    z2 = engine.conv2d(y, engine.pack_weight(w1n.float()), b1n, c3, 1, relu=True)
    torch.cuda.synchronize()
    assert torch.equal(y, y0)
    assert torch.equal(z, z2)
    _close16(z, _ref_conv(y, w1n, b1n, 1, relu=True))
