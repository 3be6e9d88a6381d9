"""GPU tests of the TMA-store epilogue of the fp16 convolution (conv_gemm_kernel<64|128|256, kOpF16>): each 64-column
chunk of a tile goes through a swizzled staging chunk in shared memory (stmatrix) and leaves with one bulk tensor store,
clipped at the output's edges by the tensor map; a mode-0 residual comes through the operand ring by TMA.  Every case runs
the same launch twice in one process, with the TMA path (odtk_set_tma_store(1), the default) and with the direct stores
(odtk_set_tma_store(0)), and requires byte-identical outputs -- including everything outside the written rectangle,
which is pre-filled with a sentinel -- and the plan to report the path it took."""
import ctypes

import pytest
import torch

from retinanet_examples_b200 import _lib, engine
from retinanet_examples_b200.model import Model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENTINEL = -1234.0   # exact in fp16


def _rand(shape, g, scale=1.0):
    return (torch.randn(shape, generator=g) * scale).to(torch.float16).to(DEV)


def _both(fn, budget=0):
    """fn() on the TMA path and on the direct path, under a launch budget of `budget` SMs (0: the whole device; a small
    budget makes a small shape choose the 256-wide tile).  Returns (tma result, direct result, plan of the TMA launch)."""
    L = _lib.lib()
    L.odtk_set_sm_budget(budget)
    prev = L.odtk_set_tma_store(1)
    try:
        y1 = fn()
        p1 = engine.last_plan()
        assert L.odtk_set_tma_store(0) == 1
        y0 = fn()
        p0 = engine.last_plan()
        torch.cuda.synchronize()
    finally:
        L.odtk_set_tma_store(prev)
        L.odtk_set_sm_budget(0)
    assert p0["tma_store"] == 0 and p0["bn"] == p1["bn"], (p0, p1)
    return y1, y0, p1


def _budgets(m_tiles, cout):
    """Launch budgets that select N tiles 64 (if Cout allows), 128 and 256 for a launch of m_tiles M tiles."""
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    n128 = m_tiles * ((cout + 127) // 128)
    return sorted({2, min(n128, sms) & ~1, min(n128 + 1, sms)} - {0, 1})


def _sentinel_out(shape):
    return torch.full(shape, SENTINEL, dtype=torch.float16, device=DEV)


# mode 0 (1x1): M = n*h*w not a multiple of 128; Cout 720 and 192 end inside a 64-column chunk
@pytest.mark.parametrize("n,h,w,cin,cout", [(2, 27, 29, 256, 512), (2, 19, 27, 128, 720), (1, 61, 53, 256, 192),
                                            (3, 11, 13, 64, 64)])
@pytest.mark.parametrize("with_res", [False, True])
def test_mode0_ragged_m_every_tile_width(n, h, w, cin, cout, with_res):
    g = torch.Generator().manual_seed(n * 5 + h * 3 + w + cin + cout + with_res)
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, 1, 1), g, 0.05), torch.randn(cout, generator=g).to(DEV)
    res = _rand((n, h, w, cout), g) if with_res else None
    pw = engine.pack_weight(wt.float())
    seen = set()
    for budget in _budgets((n * h * w + 127) // 128, cout):
        y1, y0, plan = _both(lambda: engine.conv2d(x, pw, b, cout, 1, relu=True, residual=res), budget)
        assert plan["tma_store"] == 1 and plan["mode"] == 0, plan
        assert torch.equal(y1, y0), (budget, plan["bn"])
        seen.add(plan["bn"])
    assert {128, 256} <= seen or cout <= 128, seen


def test_mode0_residual_row_stride_and_relu6():
    """A residual with a row stride wider than Cout (ldr) through the ring, ReLU6, and a Cout of 64 (BN 64)."""
    g = torch.Generator().manual_seed(9)
    n, h, w, cin = 1, 37, 41, 128
    for cout in (64, 256):
        x, wt = _rand((n, h, w, cin), g), _rand((cout, cin, 1, 1), g, 0.05)
        b = torch.randn(cout, generator=g).to(DEV)
        big = _rand((n, h, w, cout + 64), g)
        pw = engine.pack_weight(wt.float())

        def run():
            y = torch.empty((n, h, w, cout), dtype=torch.float16, device=DEV)
            d = engine.ConvDesc()
            d.x, d.w, d.bias, d.residual, d.y = x.data_ptr(), pw.data_ptr(), b.data_ptr(), big.data_ptr(), y.data_ptr()
            d.n, d.h, d.width, d.cin, d.cout, d.ksize, d.relu = n, h, w, cin, cout, 1, 2
            d.out_mode, d.ldy, d.ldr, d.stride, d.groups = engine.OUT_NHWC_F16, 0, cout + 64, 1, 1
            _lib.check(_lib.lib().odtk_conv2d(ctypes.byref(d), engine._stream()), "conv2d")
            return y
        y1, y0, plan = _both(run)
        assert plan["tma_store"] == 1
        assert torch.equal(y1, y0)


def test_mode0_output_row_stride_wider_than_cout():
    """ldy > Cout: the columns between Cout and ldy keep their sentinel."""
    g = torch.Generator().manual_seed(11)
    n, h, w, cin, cout, ldy = 2, 23, 31, 128, 192, 264
    x, b = _rand((n, h, w, cin), g), torch.randn(cout, generator=g).to(DEV)
    for ks in (1, 3):
        pw = engine.pack_weight(_rand((cout, cin, ks, ks), g, 0.03).float())

        def run():
            y = _sentinel_out((n, h, w, ldy))
            d = engine.ConvDesc()
            d.x, d.w, d.bias, d.y = x.data_ptr(), pw.data_ptr(), b.data_ptr(), y.data_ptr()
            d.n, d.h, d.width, d.cin, d.cout, d.ksize, d.relu = n, h, w, cin, cout, ks, 1
            d.out_mode, d.ldy, d.ldr, d.stride, d.groups = engine.OUT_NHWC_F16, ldy, 0, 1, 1
            _lib.check(_lib.lib().odtk_conv2d(ctypes.byref(d), engine._stream()), "conv2d")
            return y
        y1, y0, plan = _both(run)
        assert plan["tma_store"] == 1
        assert torch.equal(y1, y0)
        assert bool((y1[..., cout:] == SENTINEL).all())


# mode 1 (dense 3x3): patches that do not divide the image, odd sizes
@pytest.mark.parametrize("n,h,w,cin,cout", [(2, 29, 43, 256, 512), (1, 27, 45, 128, 720), (4, 21, 37, 64, 256),
                                            (1, 7, 130, 64, 128)])
def test_mode1_dense_partial_patches(n, h, w, cin, cout):
    g = torch.Generator().manual_seed(n * 7 + h + w + cin + cout)
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, 3, 3), g, 0.03), torch.randn(cout, generator=g).to(DEV)
    pw = engine.pack_weight(wt.float())
    for budget in (2, 0):
        y1, y0, plan = _both(lambda: engine.conv2d(x, pw, b, cout, 3, relu=True), budget)
        assert plan["tma_store"] == 1 and plan["mode"] == 1, plan
        assert torch.equal(y1, y0), plan["bn"]
    # a residual on a spatial tile stays on the direct path
    res = _rand((n, h, w, cout), g)
    y1, y0, plan = _both(lambda: engine.conv2d(x, pw, b, cout, 3, residual=res))
    assert plan["tma_store"] == 0
    assert torch.equal(y1, y0)


@pytest.mark.parametrize("n,h,w,cin,cout,ks", [(2, 31, 45, 128, 256, 3), (1, 33, 27, 256, 512, 1),   # odd: mode 1 s2
                                               (2, 40, 58, 128, 256, 3), (1, 26, 34, 256, 1024, 1)])  # even: mode 3
def test_stride2(n, h, w, cin, cout, ks):
    g = torch.Generator().manual_seed(n * 3 + h + w * 5 + cin + cout + ks)
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, ks, ks), g, 0.03), torch.randn(cout, generator=g).to(DEV)
    pw = engine.pack_weight(wt.float())
    for budget in (2, 0):
        y1, y0, plan = _both(lambda: engine.conv2d(x, pw, b, cout, ks, relu=True, stride=2), budget)
        assert plan["tma_store"] == 1 and plan["mode"] == (1 if h % 2 else 3), plan
        assert torch.equal(y1, y0), plan["bn"]


def test_fpn_upsample_addend():
    g = torch.Generator().manual_seed(21)
    n, h, w, cin, cout = 2, 26, 38, 512, 256
    x, wt, b = _rand((n, h, w, cin), g), _rand((cout, cin, 1, 1), g, 0.05), torch.randn(cout, generator=g).to(DEV)
    up = _rand((n, h // 2, w // 2, cout), g)
    pw = engine.pack_weight(wt.float())
    for budget in _budgets((n * h * w + 127) // 128, cout):
        y1, y0, plan = _both(lambda: engine.conv2d(x, pw, b, cout, 1, upsample=up), budget)
        assert plan["tma_store"] == 1
        assert torch.equal(y1, y0), plan["bn"]


def _atlas(n):
    sizes = ((100, 160), (50, 80), (25, 40), (13, 20), (7, 10))
    at = Model("ResNet18FPN", classes=4)._atlas_for(n, sizes, torch.device(DEV))
    valid = torch.zeros((at["ha"], at["wa"]), dtype=torch.bool, device=DEV)
    for r, (h, w) in zip(at["rows"], sizes):
        valid[r:r + h, :w] = True
    x = _rand((n, at["ha"], at["wa"], 256), torch.Generator().manual_seed(n))
    x[:, ~valid] = 0
    return at, sizes, valid, x


def test_level_view_output_keeps_the_rest():
    """A level-view output (oR, oW > W): nothing outside the level's rectangle changes."""
    at, sizes, valid, x = _atlas(1)
    g = torch.Generator().manual_seed(4)
    r, (h, w) = at["rows"][1], sizes[1]
    lvl = x[:, r:r + h, :w].contiguous()
    for cout in (256, 128):
        pw = engine.pack_weight(_rand((cout, 256, 3, 3), g, 0.03).float())
        b = torch.randn(cout, generator=g).to(DEV)

        def run():
            y = _sentinel_out((1, 2 * h + 9, at["wa"] + 32, cout))
            engine.conv2d(lvl, pw, b, cout, 3, relu=True, out=engine.AtlasView(y, h + 9, h, w))
            return y
        for budget in (2, 0):
            y1, y0, plan = _both(run, budget)
            assert plan["tma_store"] == 1
            assert torch.equal(y1, y0)
            outside = torch.ones(y1.shape[1:3], dtype=torch.bool, device=DEV)
            outside[h + 9:2 * h + 9, :w] = False
            assert bool((y1[:, outside] == SENTINEL).all())


def test_atlas_tile_table_batch2():
    """A head tower layer over a whole 800 x 1280 atlas through its tile table, batch 2: tiles inside a level take the TMA
    path, tiles clipped by a level's edge the direct one; gap rows and columns stay exactly zero."""
    at, sizes, valid, x = _atlas(2)
    g = torch.Generator().manual_seed(3)
    wt, b = _rand((256, 256, 3, 3), g, 0.03), torch.randn(256, generator=g).to(DEV)
    pw = engine.pack_weight(wt.float())

    def tower():
        y = torch.zeros_like(x)
        engine.conv2d(x, pw, b, 256, 3, relu=True, out=y, tile_tab=at["tab"])
        return y
    for budget in (2, 0):
        y1, y0, plan = _both(tower, budget)
        assert plan["tma_store"] == 1
        assert torch.equal(y1, y0)
        assert int((y1[:, ~valid] != 0).sum()) == 0


def _tail_args(n, h, w, c1, c2, g, proj=False):
    x = _rand((n, h, w, c1), g)
    w2, b2 = _rand((c1, c1, 3, 3), g, 0.04), torch.randn(c1, generator=g).to(DEV) * 0.5
    w3, b3 = _rand((c2, c1, 1, 1), g, 0.08), torch.randn(c2, generator=g).to(DEV) * 0.5
    res = None if proj else _rand((n, h, w, c2), g)
    return (x, engine.pack_weight(w2.float()), b2, engine.pack_weight(w3.float()), b3, res)


@pytest.mark.parametrize("n,h,w,c1,c3,proj", [(2, 23, 29, 64, 0, False), (1, 19, 37, 64, 0, True), (2, 13, 27, 64, 64, False),
                                              (1, 29, 21, 64, 128, False), (2, 17, 31, 128, 0, False)])
def test_bottleneck_tail_y_and_z(n, h, w, c1, c3, proj):
    """The four tail instances <C1, N3> = <64, 0> (with and without the projected identity), <64, 64>, <64, 128> and
    <128, 0>, at sizes whose patches do not divide the image: y and z byte-identical between the two paths."""
    c2 = 4 * c1
    g = torch.Generator().manual_seed(n * 3 + h * 5 + w + c1 + c3)
    args = _tail_args(n, h, w, c1, c2, g, proj)
    kw = dict(relu=True)
    if proj:
        kw.update(xproj=_rand((n, h, w, 64), g), wproj=engine.pack_weight(_rand((c2, 64, 1, 1), g, 0.1).float()))
    if c3:
        kw.update(w_next=engine.pack_weight(_rand((c3, c2, 1, 1), g, 0.06).float()), b_next=torch.randn(c3, generator=g).to(DEV))
    L = _lib.lib()
    prev = L.odtk_set_tma_store(1)
    try:
        on = engine.bottleneck_tail(*args, **kw)
        L.odtk_set_tma_store(0)
        off = engine.bottleneck_tail(*args, **kw)
        torch.cuda.synchronize()
    finally:
        L.odtk_set_tma_store(prev)
    on, off = (on, off) if c3 else ((on,), (off,))
    for a, b in zip(on, off):
        assert torch.equal(a, b)
