"""GPU tests of the INT8 network scope: the new s8 convolution paths (stride 2, residual, upsample-add, output into an atlas
view) bit-exact against a CPU emulation, the ReLU copy of an s8 atlas level, and the model's network-scope heads
bit-identical to tests/int8_network_oracle.py from the model's own quantised C3, plus detections, match rate and plumbing
(CUDA graphs, parallel heads, format-2 tables, switching scope and precision, training mode, unsupported backbones)."""
import ctypes
import json

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import int8_network_oracle as net_oracle
import int8_oracle
from oracle import model_ref
from retinanet_examples_b200 import _lib, calib, engine
from retinanet_examples_b200.model import Model, make_state_dict
from test_int8_network_host import MATCH_NETWORK_ORACLE, match, spread_head

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
E_UNSUPPORTED = -3


def _rand_s8(shape, seed):
    return torch.randint(-127, 128, shape, dtype=torch.int8, generator=torch.Generator().manual_seed(seed))


def _layer(cin, cout, ks, seed, s_in=0.05):
    g = torch.Generator().manual_seed(seed)
    wq, s_w = engine.pack_weight_s8(torch.randn((cout, cin, ks, ks), generator=g) * 0.02)
    alpha = s_w * torch.tensor(s_in, dtype=torch.float32)
    return wq.to(DEV), alpha.to(DEV), (torch.randn(cout, generator=g) * 0.5).to(DEV)


def _emulate(xq, wq, alpha, bias, ks, stride, relu, inv_out, res=None, rs=0.0, up=None, us=0.0):
    """CPU emulation of odtk_conv2d_s8_ex with an NHWC s8 output (inv_out None: the fp32 values before requantisation)."""
    cout, cin = wq.shape[0], xq.shape[3]
    acc = F.conv2d(xq.permute(0, 3, 1, 2).double(), wq.cpu().view(cout, ks, ks, cin).permute(0, 3, 1, 2).double(),
                   stride=stride, padding=ks // 2)
    y = int8_oracle.fmaf(acc, alpha.cpu(), bias.cpu())
    if res is not None:
        y = net_oracle.fma_add(res.permute(0, 3, 1, 2).double(), torch.tensor(rs, dtype=torch.float32), y)
    if up is not None:
        y = net_oracle.fma_add(net_oracle.upsample2(up.permute(0, 3, 1, 2).double()), torch.tensor(us, dtype=torch.float32), y)
    if relu:
        y = F.relu(y)
    if inv_out is None:
        return y
    return torch.round(y * torch.tensor(inv_out, dtype=torch.float32)).clamp(-127, 127).to(torch.int8).permute(0, 2, 3, 1)


@pytest.mark.parametrize("n,h,w,cin,cout,ks,stride,extra,mode", [
    (2, 32, 48, 256, 256, 3, 2, None, 3),          # layer3/4 block-0 3x3, even: parity split
    (2, 32, 48, 512, 1024, 1, 2, None, 3),         # block-0 downsample 1x1, even
    (8, 8, 12, 512, 256, 3, 2, None, 3),           # pyramid6 on an even C5
    (2, 25, 40, 512, 256, 3, 2, None, 1),          # pyramid6 on an odd C5: element-strided boxes
    (2, 13, 20, 256, 256, 3, 2, None, 1),          # pyramid7 on an odd P6
    (2, 25, 39, 256, 512, 1, 2, None, 1),          # 1x1 stride 2, odd
    (2, 32, 48, 256, 1024, 1, 1, "res", 0),        # bottleneck conv3 + identity
    (2, 16, 24, 256, 256, 3, 1, "res", 1),         # basic-block conv2 + identity
    (2, 16, 24, 512, 256, 1, 1, "up", 0),          # lateral + top-down nearest-2x addend
    (1, 8, 12, 256, 256, 1, 1, "res+up", 0),       # both addends, narrow: N tile 64
])
def test_conv_s8_ex_bit_exact(n, h, w, cin, cout, ks, stride, extra, mode):
    xq = _rand_s8((n, h, w, cin), 1)
    wq, alpha, b = _layer(cin, cout, ks, 2)
    oh, ow = ((h - 1) // 2 + 1, (w - 1) // 2 + 1) if stride == 2 else (h, w)
    res = _rand_s8((n, oh, ow, cout), 3) if "res" in (extra or "") else None
    up = _rand_s8((n, oh // 2, ow // 2, cout), 4) if "up" in (extra or "") else None
    rs, us = 0.0371, 0.0213
    # output scale: the largest outputs saturate (127 * s_out is 60 % of max|y|)
    y = _emulate(xq, wq, alpha, b, ks, stride, True, None, res, rs, up, us)
    inv = float(np.float32(1.0) / np.float32(0.6 * float(y.max()) / 127))
    got = engine.conv2d_s8(xq.to(DEV), wq, alpha, b, cout, ks, relu=True, inv_out_scale=inv, stride=stride,
                           residual=res.to(DEV) if res is not None else None, res_scale=rs,
                           upsample=up.to(DEV) if up is not None else None, up_scale=us).cpu()
    plan = engine.last_plan()
    assert plan["mode"] == mode, plan
    ref = _emulate(xq, wq, alpha, b, ks, stride, True, inv, res, rs, up, us)
    assert got.shape == ref.shape and torch.equal(got, ref)
    assert int((got == 127).sum()) > 0 and int((got == 0).sum()) > 0


def test_conv_s8_ex_level_views_and_n_tiles():
    """Stride-2 input from a level view of an s8 atlas (element-strided boxes), outputs into level views of another atlas
    (stride 1 and 2); gap rows / columns stay untouched; both N tiles."""
    m = Model("ResNet18FPN", classes=6)
    sizes = ((64, 96), (32, 48), (16, 24), (8, 12), (4, 6))
    at = m._atlas_for(2, sizes, torch.device(DEV))
    x = _rand_s8((2, at["ha"], at["wa"], 256), 5).to(DEV)
    y = torch.zeros((2, at["ha"], at["wa"], 256), dtype=torch.int8, device=DEV)
    wq, alpha, b = _layer(256, 256, 3, 6)
    inv = float(np.float32(1.0) / np.float32(0.09))
    seen = set()
    for src, dst, stride in ((1, 2, 2), (3, 4, 2), (0, 0, 1), (2, 2, 1)):
        (hs, ws), (hd, wd) = sizes[src], sizes[dst]
        vin = engine.AtlasView(x, at["rows"][src], hs, ws)
        vout = engine.AtlasView(y, at["rows"][dst], hd, wd)
        engine.conv2d_s8(vin, wq, alpha, b, 256, 3, relu=True, out=vout, inv_out_scale=inv, stride=stride)
        plan = engine.last_plan()
        assert plan["mode"] == 1, plan
        seen.add(plan["bn"])
        ref = _emulate(vin.dense().cpu(), wq, alpha, b, 3, stride, True, inv)
        assert torch.equal(vout.dense().cpu(), ref), (src, dst)
    valid = torch.zeros((at["ha"], at["wa"]), dtype=torch.bool)
    for r, (h, w) in zip(at["rows"], sizes):
        valid[r:r + h, :w] = True
    assert int(y.cpu()[:, ~valid].abs().max()) == 0
    assert seen == {64, 128}


def test_relu_from_view_s8():
    x = _rand_s8((2, 30, 16, 256), 7).to(DEV)
    v = engine.AtlasView(x, 17, 7, 10)
    got = engine.relu_from_view_s8(v).cpu()
    assert torch.equal(got, v.dense().cpu().clamp(min=0))


def _desc(xq, wq, alpha, y, n, h, w, cin, cout, ks):
    d = engine.ConvS8Desc()
    d.x, d.w, d.alpha, d.y = xq.data_ptr(), wq.data_ptr(), alpha.data_ptr(), y.data_ptr()
    d.n, d.h, d.width, d.cin, d.cout, d.ksize, d.relu, d.out_mode, d.inv_out_scale = n, h, w, cin, cout, ks, 1, engine.OUT_NHWC_S8, 0.1
    return d


def test_conv_s8_zeroed_extension_identical_and_unsupported_combinations():
    lib = _lib.lib()
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    xq = _rand_s8((2, 16, 24, 256), 8).to(DEV)
    wq, alpha, b = _layer(256, 256, 3, 9)
    y0, y1 = torch.empty_like(xq), torch.full_like(xq, 5)
    d = _desc(xq, wq, alpha, y0, 2, 16, 24, 256, 256, 3)
    assert lib.odtk_conv2d_s8(ctypes.byref(d), st) == 0
    e = engine.ConvS8ExDesc()
    e.base = _desc(xq, wq, alpha, y1, 2, 16, 24, 256, 256, 3)
    assert lib.odtk_conv2d_s8_ex(ctypes.byref(e), st) == 0
    torch.cuda.synchronize()
    assert torch.equal(y0, y1)
    tab = torch.zeros((4, 4), dtype=torch.int32, device=DEV)

    def rc(**kw):
        e = engine.ConvS8ExDesc()
        e.base = _desc(xq, wq, alpha, y1, 2, 16, 24, 256, 256, kw.pop("ks", 3))
        for k, v in kw.items():
            setattr(e.base if hasattr(e.base, k) else e, k, v)
        return lib.odtk_conv2d_s8_ex(ctypes.byref(e), st)

    assert rc(residual=y0.data_ptr(), tile_tab=tab.data_ptr(), tab_tiles=4) == E_UNSUPPORTED     # addend + tile table
    assert rc(upsample=y0.data_ptr(), y_rows=40, y_width=24) == E_UNSUPPORTED                   # addend + output view
    assert rc(residual=y0.data_ptr(), out_mode=engine.OUT_NCHW_F32) == E_UNSUPPORTED            # addend, fp32 output
    assert rc(y_rows=40, y_width=24, ks=1) == E_UNSUPPORTED                                     # output view, 1x1
    assert rc(upsample=y0.data_ptr(), stride=2) == E_UNSUPPORTED                                # upsample, stride 2
    assert rc(relu=2) == E_UNSUPPORTED                                                          # ReLU6
    assert rc(stride=3) == E_UNSUPPORTED
    assert rc(cin=192, residual=y0.data_ptr()) == E_UNSUPPORTED                                 # cin % 128
    torch.cuda.synchronize()


# ---- the model in network scope ---------------------------------------------------------------------------------------
def _net_model(backbone, classes, rotated, shape, seed=10):
    na = 27 if rotated else 9
    sd = spread_head(make_state_dict(backbone, classes, na, rotated, seed))
    x = torch.randn(shape, generator=torch.Generator().manual_seed(4))
    m = Model(backbone, classes=classes, rotated_bbox=rotated).load_state_dict(sd).cuda()
    table = m.calibrate([x], scope="network")
    m.set_precision("int8", table, scope="network")
    return m, x.to(DEV), table


def _forward_capturing_c3(m, x, monkeypatch):
    """forward_heads(sigmoid=False), capturing the s8 C3 the model quantised (its only fp16 -> s8 launch)."""
    seen = []
    orig = engine.quantize_f16_s8

    def spy(t, inv, out=None):
        q = orig(t, inv, out)
        seen.append(q)
        return q

    monkeypatch.setattr(engine, "quantize_f16_s8", spy)
    cls, box = m.forward_heads(x, sigmoid=False)
    monkeypatch.setattr(engine, "quantize_f16_s8", orig)
    assert len(seen) == 1
    return cls, box, seen[0].permute(0, 3, 1, 2).cpu().double()


@pytest.mark.parametrize("backbone,classes,rotated,shape", [
    ("ResNet18FPN", 6, False, (2, 3, 256, 384)), ("ResNet18FPN", 6, True, (2, 3, 256, 384)),
    ("ResNet50FPN", 6, False, (2, 3, 256, 384)), ("ResNet50FPN", 6, True, (1, 3, 256, 384)),
    ("ResNet50FPN", 80, False, (1, 3, 800, 1280)), ("ResNet101FPN", 6, False, (1, 3, 256, 384))])
def test_network_heads_bit_identical_to_oracle(backbone, classes, rotated, shape, monkeypatch):
    m, x, table = _net_model(backbone, classes, rotated, shape)
    cls, box, q3 = _forward_capturing_c3(m, x, monkeypatch)
    rc, rb = net_oracle.forward_heads(m._sd, backbone, q3, table["scales"], sigmoid=False)
    for i in range(5):
        assert torch.equal(cls[i].cpu(), rc[i]), ("cls", i)
        assert torch.equal(box[i].cpu(), rb[i]), ("box", i)


def test_network_detections_exact_on_its_heads():
    m, x, _ = _net_model("ResNet18FPN", 6, False, (2, 3, 256, 384))
    scores, boxes, cl = [t.clone().cpu().numpy() for t in m(x)]
    assert (scores > 0).sum() > 20
    cls_h, box_h = m.forward_heads(x)
    (os_, ob, oc), _ = model_ref.postprocess([c.cpu() for c in cls_h], [b.cpu() for b in box_h], x.shape[-1])
    np.testing.assert_array_equal(scores, os_)
    np.testing.assert_array_equal(cl, oc)
    np.testing.assert_allclose(boxes, ob, atol=1e-3, rtol=0)


@pytest.mark.parametrize("backbone", ["ResNet18FPN", "ResNet50FPN"])
def test_network_vs_fp16_detection_match_rate(backbone):
    """The oracle's network-scope rate (test_int8_network_host.MATCH_NETWORK_ORACLE) minus 5 points for the fp16 rounding
    differences between the product's and the oracle's stem / layer1 / layer2."""
    m, x, _ = _net_model(backbone, 6, False, (2, 3, 256, 384))
    got = [t.clone().cpu().numpy() for t in m(x)]
    m.set_precision("fp16")
    ref = [t.cpu().numpy() for t in m(x)]
    hit = n = 0
    for img in range(x.shape[0]):
        h, k = match([t[img] for t in got], [t[img] for t in ref])
        hit, n = hit + h, n + k
    assert n > 20
    assert hit / n >= MATCH_NETWORK_ORACLE[backbone] - 0.05, (hit, n)


def test_network_graph_replay_parallel_heads_and_fresh_model_from_table(tmp_path):
    m, x, table = _net_model("ResNet18FPN", 6, False, (2, 3, 256, 384))
    x2 = torch.randn((2, 3, 256, 384), generator=torch.Generator().manual_seed(5)).to(DEV)
    eager = [[t.clone() for t in m(v)] for v in (x, x2)]
    m.parallel_heads = False
    for a, b in zip(m(x), eager[0]):
        assert torch.equal(a, b)
    m.parallel_heads = True
    m.enable_cuda_graph()
    for v, e in ((x, eager[0]), (x2, eager[1]), (x, eager[0])):
        for a, b in zip(m(v), e):
            assert torch.equal(a, b)
    m.enable_cuda_graph(False)
    path = str(tmp_path / "net.json")
    table2 = m.calibrate([x.cpu()], table=path, scope="network")
    assert table2 == table and json.load(open(path))["format"] == 2
    fresh = Model("ResNet18FPN", classes=6).load_state_dict(m._sd).cuda().set_precision("int8", path, scope="network")
    for a, b in zip(fresh(x), eager[0]):
        assert torch.equal(a, b)


def test_calibration_tables_and_switching_scope_and_precision():
    """The network table's 9 head scales are the heads table's; calibrate() with default arguments gives the format-1
    heads table; network -> heads -> fp16 gives exactly what freshly configured models give; training stays fp16."""
    m, x, table = _net_model("ResNet18FPN", 6, False, (2, 3, 256, 384))
    heads = m.calibrate([x.cpu()])
    assert heads["format"] == 1 and "scope" not in heads and set(heads["scales"]) == set(calib.TENSORS)
    assert {k: table["scales"][k] for k in calib.TENSORS} == heads["scales"]
    net_out = [t.clone() for t in m(x)]

    def fresh(precision="fp16", tbl=None, scope="heads"):
        f = Model("ResNet18FPN", classes=6).load_state_dict(m._sd).cuda()
        return f.set_precision(precision, tbl, scope) if precision != "fp16" else f

    for a, b in zip(net_out, fresh("int8", table, "network")(x)):
        assert torch.equal(a, b)
    m.set_precision("int8", heads)
    heads_out = [t.clone() for t in m(x)]
    assert not all(torch.equal(a, b) for a, b in zip(heads_out, net_out))
    for a, b in zip(heads_out, fresh("int8", heads)(x)):
        assert torch.equal(a, b)
    m.set_precision("int8", table, scope="network")
    targets = torch.tensor([[[20., 30., 120., 140., 1.], [200., 40., 300., 200., 3.]]] * 2).to(DEV)
    plain = fresh()
    m.train(); plain.train()
    for a, b in zip(m([x, targets]), plain([x, targets])):
        assert torch.equal(a, b)
    m.eval(); plain.eval()
    m.set_precision("fp16")
    for a, b in zip(m(x), plain(x)):
        assert torch.equal(a, b)
    with pytest.raises(ValueError):
        m.set_precision("int8", heads, scope="network")              # a format-1 table
    with pytest.raises(ValueError):
        m.set_precision("int8", table, scope="everything")


@pytest.mark.parametrize("backbone", ["ResNeXt50_32x4dFPN", "MobileNetV2FPN"])
def test_unsupported_backbones_reject_network_scope(backbone):
    m = Model(backbone, classes=4).load_state_dict(make_state_dict(backbone, 4, 9, False, 1)).cuda()
    x = torch.randn((1, 3, 128, 256), generator=torch.Generator().manual_seed(2))
    with pytest.raises(ValueError):
        m.calibrate([x], scope="network")
    heads = m.calibrate([x])
    with pytest.raises(ValueError):
        m.set_precision("int8", heads, scope="network")
    m.set_precision("int8", heads)
    m(x.to(DEV))
