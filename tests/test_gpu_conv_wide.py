"""GPU tests of the 128 x 256 fp16 convolution tile (conv_gemm_kernel<256, kOpF16>): the host selects it for wide layers
with many tiles, so the shapes here are small and the launch budget (odtk_set_sm_budget) is lowered until the rule picks
it.  Every case checks the plan, a CUDA fp32 torch convolution of the same fp16 operands (TF32 off) within the fp16 bound
of test_gpu_conv.py, and that the same launch on 128-wide N tiles gives the same bits: both tiles run the same K blocks
and k16 steps in the same order."""
import pytest
import torch
import torch.nn.functional as F

from retinanet_examples_b200 import _lib, engine
from retinanet_examples_b200.model import Model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WIDE_BUDGET = 2   # SMs: a few dozen 256-wide tiles fill the waves the rule asks for


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
    """fn() under a launch budget of `sms` SMs (0: the whole device); returns its result and the plan of its launch."""
    _lib.lib().odtk_set_sm_budget(sms)
    try:
        out = fn()
        plan = engine.last_plan()
        torch.cuda.synchronize()
    finally:
        _lib.lib().odtk_set_sm_budget(0)
    return out, plan


def _wide_and_narrow(fn, cout):
    """fn() at N tile 256, then again on a budget where the rule keeps 128-wide tiles; both results."""
    y256, plan = _with_budget(WIDE_BUDGET, fn)
    assert plan["bn"] == 256 and plan["num_n_tiles"] == (cout + 255) // 256, plan
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    budget = min(plan["num_m_tiles"] * ((cout + 127) // 128), sms) & ~1
    y128, plan = _with_budget(budget, fn)
    assert plan["bn"] == 128, plan
    return y256, y128


@pytest.mark.parametrize("n,h,w,cin,cout,ks,relu", [
    (1, 48, 64, 256, 256, 3, 1), (2, 24, 32, 256, 512, 3, 0), (1, 32, 32, 256, 1024, 3, 2), (1, 16, 32, 256, 2048, 3, 1),
    (1, 33, 47, 128, 720, 3, 0), (1, 48, 64, 256, 1024, 1, 1), (1, 16, 32, 512, 2048, 1, 0), (1, 25, 39, 256, 720, 1, 2)])
def test_wide_tile_dense(n, h, w, cin, cout, ks, relu):
    """Dense 3x3 (shifted boxes, ragged patches) and 1x1 (GEMM rows, ragged last M tile); Cout 256 ... 2048 and 720 (two
    full tiles and 208 columns: zero-filled weight rows, columns that are not stored); ReLU / ReLU6."""
    g = torch.Generator().manual_seed(n * 7 + h + w + cin + cout + ks)
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, ks, ks), g, 0.03), torch.randn(cout, generator=g).to(DEV)
    pw = engine.pack_weight(wt.float())
    y256, y128 = _wide_and_narrow(lambda: engine.conv2d(x, pw, b, cout, ks, relu=relu), cout)
    assert torch.equal(y256, y128)
    _close16(y256, _ref_conv(x, wt, b, ks, relu=relu))


@pytest.mark.parametrize("ks", [1, 3])
def test_wide_tile_residual_and_upsample_addends(ks):
    g = torch.Generator().manual_seed(40 + ks)
    n, h, w, cin, cout = 2, 26, 48, 256, 512
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, ks, ks), g, 0.03), torch.randn(cout, generator=g).to(DEV)
    res, up = _rand((n, h, w, cout), g), _rand((n, h // 2, w // 2, cout), g)
    pw = engine.pack_weight(wt.float())
    y256, y128 = _wide_and_narrow(lambda: engine.conv2d(x, pw, b, cout, ks, relu=True, residual=res), cout)
    assert torch.equal(y256, y128)
    _close16(y256, _ref_conv(x, wt, b, ks, relu=True, residual=res))
    y256, y128 = _wide_and_narrow(lambda: engine.conv2d(x, pw, b, cout, ks, upsample=up), cout)
    assert torch.equal(y256, y128)
    _close16(y256, _ref_conv(x, wt, b, ks, upsample=up))


@pytest.mark.parametrize("cout,mode", [(720, engine.OUT_NCHW_F32_SIGMOID), (720, engine.OUT_NCHW_F32), (512, engine.OUT_NCHW_F32)])
def test_wide_tile_nchw_fp32_outputs(cout, mode):
    g = torch.Generator().manual_seed(cout + mode)
    n, h, w, cin = 2, 25, 40, 256
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, 3, 3), g, 0.02), torch.randn(cout, generator=g).to(DEV)
    pw = engine.pack_weight(wt.float())
    y256, y128 = _wide_and_narrow(lambda: engine.conv2d(x, pw, b, cout, 3, out_mode=mode), cout)
    assert torch.equal(y256, y128)
    ref = _ref_conv(x, wt, b, 3)
    if mode == engine.OUT_NCHW_F32_SIGMOID:
        ref = torch.sigmoid(ref)
    assert (y256 - ref).abs().max().item() <= 1e-4 * max(1.0, ref.abs().max().item())


def _atlas(n):
    """The pyramid atlas of an 800 x 1280 image (levels P3-P7, 182 tiles per image) and a random fp16 input in it, zero
    in the gap rows and right of the narrower levels."""
    sizes = ((100, 160), (50, 80), (25, 40), (13, 20), (7, 10))
    at = Model("ResNet18FPN", classes=4)._atlas_for(n, sizes, torch.device(DEV))
    valid = torch.zeros((at["ha"], at["wa"]), dtype=torch.bool, device=DEV)
    for r, (h, w) in zip(at["rows"], sizes):
        valid[r:r + h, :w] = True
    x = _rand((n, at["ha"], at["wa"], 256), torch.Generator().manual_seed(n))
    x[:, ~valid] = 0
    return at, sizes, valid, x


def test_wide_tile_atlas_tile_table():
    """A head tower layer: one launch over the whole atlas through its tile table; every level against its dense
    convolution, gap rows and the columns right of the narrow levels exactly zero."""
    at, sizes, valid, x = _atlas(1)
    g = torch.Generator().manual_seed(3)
    wt, b = _rand((256, 256, 3, 3), g, 0.03), torch.randn(256, generator=g).to(DEV)
    pw = engine.pack_weight(wt.float())

    def tower():
        y = torch.zeros_like(x)
        engine.conv2d(x, pw, b, 256, 3, relu=True, out=y, tile_tab=at["tab"])
        return y
    y256, y128 = _wide_and_narrow(tower, 256)
    assert torch.equal(y256, y128)
    assert int((y256[:, ~valid] != 0).sum()) == 0
    for r, (h, w) in zip(at["rows"], sizes):
        _close16(y256[:, r:r + h, :w], _ref_conv(x[:, r:r + h, :w], wt, b, 3, relu=True))


def test_wide_tile_level_views_in_and_out():
    """Final-layer geometry: a level view of the atlas in (x_rows / x_width), and a level view out (y_rows / y_width)."""
    at, sizes, valid, x = _atlas(1)
    g = torch.Generator().manual_seed(4)
    r, (h, w) = at["rows"][0], sizes[0]
    wt, b = _rand((256, 256, 3, 3), g, 0.03), torch.randn(256, generator=g).to(DEV)
    pw = engine.pack_weight(wt.float())
    ref = _ref_conv(x[:, r:r + h, :w], wt, b, 3, relu=True)

    def view_in():
        return engine.conv2d(engine.AtlasView(x, r, h, w), pw, b, 256, 3, relu=True)
    y256, y128 = _wide_and_narrow(view_in, 256)
    assert torch.equal(y256, y128)
    _close16(y256, ref)
    lvl = x[:, r:r + h, :w].contiguous()

    def view_out():   # P3-sized output at row h + 8 of a wider, taller buffer
        y = torch.zeros((1, 2 * h + 8, at["wa"] + 32, 256), dtype=torch.float16, device=DEV)
        engine.conv2d(lvl, pw, b, 256, 3, relu=True, out=engine.AtlasView(y, h + 8, h, w))
        return y
    y256, y128 = _wide_and_narrow(view_out, 256)
    assert torch.equal(y256, y128)
    assert int((y256[:, :h + 8] != 0).sum()) == 0 and int((y256[:, :, w:] != 0).sum()) == 0
    _close16(y256[:, h + 8:h + 8 + h, :w], ref)


def test_candidate_sink_keeps_128_wide_tiles():
    """Class-head final layer on the inference path (sigmoid + threshold + candidate append): its epilogue ran slower on
    256-wide tiles, so it keeps N tile 128 on budgets where the same layer with an NCHW output goes wide.  The candidates
    (in any order) are exactly the scores above the threshold of the wide NCHW sigmoid launch."""
    g = torch.Generator().manual_seed(5)
    n, h, w, cin, cout = 2, 25, 40, 256, 720
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, 3, 3), g, 0.02), (torch.randn(cout, generator=g) - 1.5).to(DEV)
    pw = engine.pack_weight(wt.float())
    cap, bins, thresh = cout * h * w, 2048, 0.3

    def launch():
        counts = torch.zeros(n, dtype=torch.int32, device=DEV)
        hist = torch.zeros((n, bins), dtype=torch.int32, device=DEV)
        cand = torch.zeros((n, cap, 2), dtype=torch.int32, device=DEV)
        sink = _lib.CandSink(counts.data_ptr(), hist.data_ptr(), cand.data_ptr(), cap, 0x3e000000, 16, bins, thresh)
        engine.conv2d(x, pw, b, cout, 3, out_mode=engine.OUT_CANDIDATES, sink=sink)
        torch.cuda.synchronize()
        return counts, hist, cand
    (counts, hist, cand), plan = _with_budget(WIDE_BUDGET, launch)
    assert plan["bn"] == 128, plan
    dense, plan = _with_budget(WIDE_BUDGET, lambda: engine.conv2d(x, pw, b, cout, 3, out_mode=engine.OUT_NCHW_F32_SIGMOID))
    assert plan["bn"] == 256, plan
    assert int(hist.sum()) == int(counts.sum())
    for i in range(n):
        k = int(counts[i])
        assert 0 < k < cap
        hit = (dense[i].flatten() > thresh).nonzero().flatten().to(torch.int32)
        assert torch.equal(cand[i, :k, 1].sort().values, hit)
