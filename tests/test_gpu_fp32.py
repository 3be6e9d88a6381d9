"""GPU tests of the full-precision mode (Model.set_precision("fp32")): split-TF32 convolutions (odtk_conv2d_f32) against a
float64 convolution of the same fp32 operands, the fp32 small kernels bit-exact, the heads against the reference's own
fp32 outputs and the fp32 CPU oracle, detections against the all-fp32 pipeline, and the behaviours the fp16 mode has.

Error model of one output of the convolution (K products, s = 3 * K / 8 MMAs accumulated into it): splitting both
operands as x = hi + lo (hi = rna_tf32(x), lo = rna_tf32(x - hi)) and dropping lo * lo leaves at most about
3 * 2^-22 |a b| per product; each MMA may add one fp32 rounding (or truncation) of the running sum.  Hence the per-element
bound (2^-20 + s * 2^-23) * sum_k |a_k b_k| (plus one fp32 rounding per epilogue add), which holds whatever order the
tensor cores add in."""
import io
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import resize_oracle
from oracle import model_ref, oracle
from retinanet_examples_b200 import engine
from retinanet_examples_b200.model import Model, make_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MEASURED = {}


def _conv64(x, w, b, stride, pad, residual=None, upsample=None, relu=False):
    """float64 NCHW reference of one convolution + addends + ReLU; also sum |a||b| (+ |addends|) per output."""
    y = F.conv2d(x, w, b, stride=stride, padding=pad)
    mag = F.conv2d(x.abs(), w.abs(), b.abs() if b is not None else None, stride=stride, padding=pad)
    for t in (residual, upsample):
        if t is not None:
            if t is upsample:
                t = t.repeat_interleave(2, 2).repeat_interleave(2, 3)
            y, mag = y + t, mag + t.abs()
    return (y.clamp_min(0) if relu else y), mag


def _check(got, ref, mag, t_ref, k, what):
    """Per-element worst-case bound and the norm-wise split bar: the error is at most 1/20 of single-pass TF32's (exact
    accumulation of tf32-rounded operands) up to K = 1152.  Beyond that the fp32 accumulation inside the tensor cores, not
    the operand rounding, dominates: it grows with the number of MMAs (s = 3 K / 8) while single-pass TF32's operand error
    grows only like sqrt(K), so at the heads' K = 2304 the bar is 1/10 (measured on the H100: 0.052 for Cout 36, 0.051 for
    Cout 720, against 0.002 - 0.027 for K <= 1152)."""
    s = 3 * ((k + 7) // 8)
    bound = (2.0 ** -20 + s * 2.0 ** -23) * mag + 2.0 ** -126
    err = (got.double() - ref).abs()
    ratio = float((err / bound).max())
    norm = float(err.norm() / max(float((t_ref - ref).norm()), 1e-300))
    MEASURED[what] = (ratio, norm)
    assert ratio <= 1.0, (what, ratio)
    assert norm <= (1.0 / 20 if k <= 1152 else 1.0 / 10), (what, norm)


def _tf32(t):
    return engine.tf32_rna(t.float()).double()


CASES = [  # (name, n, h, w, cin, cout, ksize, stride, relu, residual, upsample, out_mode)
    ("1x1", 2, 20, 24, 64, 64, 1, 1, True, False, False, engine.OUT_NHWC_F32),
    ("1x1_bn128", 4, 40, 48, 256, 512, 1, 1, True, True, False, engine.OUT_NHWC_F32),
    ("3x3", 2, 17, 23, 64, 64, 3, 1, True, True, False, engine.OUT_NHWC_F32),
    ("3x3_bn128", 4, 48, 64, 128, 256, 3, 1, False, False, False, engine.OUT_NHWC_F32),
    ("3x3_s2_even", 2, 32, 40, 64, 128, 3, 2, True, False, False, engine.OUT_NHWC_F32),
    ("3x3_s2_odd", 1, 25, 19, 96, 64, 3, 2, True, False, False, engine.OUT_NHWC_F32),
    ("1x1_s2_even", 2, 28, 20, 256, 512, 1, 2, False, False, False, engine.OUT_NHWC_F32),
    ("1x1_s2_odd", 1, 13, 15, 64, 128, 1, 2, False, False, False, engine.OUT_NHWC_F32),
    ("upsample", 2, 16, 24, 128, 256, 1, 1, False, False, True, engine.OUT_NHWC_F32),
    ("nchw_36", 2, 12, 20, 256, 36, 3, 1, False, False, False, engine.OUT_NCHW_F32),
    ("sigmoid_54", 1, 10, 14, 256, 54, 3, 1, False, False, False, engine.OUT_NCHW_F32_SIGMOID),
    ("nchw_720", 1, 8, 12, 256, 720, 3, 1, False, False, False, engine.OUT_NCHW_F32),
    ("nchw_2160", 1, 5, 7, 256, 2160, 3, 1, False, False, False, engine.OUT_NCHW_F32_SIGMOID),
    ("nchw_54", 1, 10, 14, 256, 54, 3, 1, False, False, False, engine.OUT_NCHW_F32),
    ("nchw_2160_raw", 1, 5, 7, 256, 2160, 3, 1, False, False, False, engine.OUT_NCHW_F32),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_conv_f32_vs_float64(case):
    name, n, h, w, cin, cout, ks, stride, relu, res, up, mode = case
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    x = torch.randn((n, cin, h, w), generator=g)
    wt = torch.randn((cout, cin, ks, ks), generator=g) * (2.0 / (cin * ks * ks)) ** 0.5
    b = torch.randn(cout, generator=g) * 0.1
    oh, ow = (h - 1) // stride + 1, (w - 1) // stride + 1
    r = torch.randn((n, cout, oh, ow), generator=g) if res else None
    u = torch.randn((n, cout, h // 2, w // 2), generator=g) if up else None
    hi, lo = engine.pack_weight_tf32x2(wt)
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous().to(DEV) if t is not None else None   # noqa: E731
    got = engine.conv2d_f32(nhwc(x), hi.to(DEV), lo.to(DEV), b.to(DEV), cout, ks, relu=relu, residual=nhwc(r), upsample=nhwc(u),
                            out_mode=mode, stride=stride)
    if "bn128" in name:
        assert engine.last_plan()["bn"] == 128
    got = got.cpu() if mode != engine.OUT_NHWC_F32 else got.permute(0, 3, 1, 2).cpu()
    d = lambda t: t.double() if t is not None else None   # noqa: E731
    ref, mag = _conv64(d(x), d(wt), d(b), stride, ks // 2, d(r), d(u), relu)
    t_ref, _ = _conv64(_tf32(x), _tf32(wt), d(b), stride, ks // 2, d(r), d(u), relu)
    if mode == engine.OUT_NCHW_F32_SIGMOID:
        ref, t_ref = torch.sigmoid(ref), torch.sigmoid(t_ref)
        # the epilogue's sigmoid is the fp16 mode's (__expf / __fdividef): 1.5e-5 absolute measured
        assert float((got.double() - ref).abs().max()) < 5e-5
        return
    _check(got, ref, mag, t_ref, ks * ks * cin, name)


@pytest.mark.parametrize("h,w", [(64, 96), (37, 51)])
def test_stem_f32_vs_float64(h, w):
    g = torch.Generator().manual_seed(h)
    x = torch.randn((2, 3, h, w), generator=g)
    wt = torch.randn((64, 3, 7, 7), generator=g) * 0.1
    b = torch.randn(64, generator=g) * 0.1
    xp = engine.pad_input_f32(x.permute(0, 2, 3, 1).contiguous().to(DEV))
    hi, lo = engine.pack_stem_weight_tf32x2(wt)
    got = engine.stem_conv_f32(xp, h, w, hi.to(DEV), lo.to(DEV), b.to(DEV), 64, relu=True)
    assert engine.last_plan()["mode"] == 2
    ref, mag = _conv64(x.double(), wt.double(), b.double(), 2, 3, relu=True)
    t_ref, _ = _conv64(_tf32(x), _tf32(wt), b.double(), 2, 3, relu=True)
    _check(got.permute(0, 3, 1, 2).cpu(), ref, mag, t_ref, 147, "stem_%dx%d" % (h, w))


def test_atlas_tile_table_and_level_views_vs_float64():
    """One launch over every level of an fp32 atlas (tile table), a 3x3 from a level view into a level view, and a stride-2
    3x3 into a level view (pyramid6), each against float64 convolutions of the dense levels."""
    m = Model("ResNet18FPN", classes=2)
    sizes = ((20, 32), (10, 16), (5, 8), (3, 4), (2, 2))
    at = m._atlas_for(2, sizes, torch.device(DEV))
    g = torch.Generator().manual_seed(7)
    atlas = torch.zeros(at["buf"][0].shape, dtype=torch.float32)
    levels = []
    for r0, (lh, lw) in zip(at["rows"], sizes):
        lv = torch.randn((2, lh, lw, 256), generator=g)
        atlas[:, r0:r0 + lh, :lw] = lv
        levels.append(lv)
    wt = torch.randn((64, 256, 3, 3), generator=g) * 0.03
    b = torch.randn(64, generator=g) * 0.1
    hi, lo = [t.to(DEV) for t in engine.pack_weight_tf32x2(wt)]
    xa, ya = atlas.to(DEV), torch.zeros(atlas.shape[:3] + (64,), dtype=torch.float32, device=DEV)
    engine.conv2d_f32(xa, hi, lo, b.to(DEV), 64, 3, relu=True, out=ya, tile_tab=at["tab"])
    ya = ya.cpu()
    for l, (r0, (lh, lw)) in enumerate(zip(at["rows"], sizes)):
        x64 = levels[l].permute(0, 3, 1, 2).double()
        ref, mag = _conv64(x64, wt.double(), b.double(), 1, 1, relu=True)
        t_ref, _ = _conv64(_tf32(x64), _tf32(wt), b.double(), 1, 1, relu=True)
        _check(ya[:, r0:r0 + lh, :lw].permute(0, 3, 1, 2), ref, mag, t_ref, 2304, "atlas_level%d" % l)
    # gap rows / columns stay zero
    mask = torch.ones(ya.shape[1:3], dtype=torch.bool)
    for r0, (lh, lw) in zip(at["rows"], sizes):
        mask[r0:r0 + lh, :lw] = False
    assert float(ya[:, mask].abs().max()) == 0.0
    # level view -> level view (stride 1), and P5 dense -> level 3 view (stride 2)
    out = torch.zeros(atlas.shape[:3] + (64,), dtype=torch.float32, device=DEV)
    src = engine.AtlasView(xa, at["rows"][1], *sizes[1])
    engine.conv2d_f32(src, hi, lo, b.to(DEV), 64, 3, out=engine.AtlasView(out, at["rows"][1], *sizes[1]))
    x64 = levels[1].permute(0, 3, 1, 2).double()
    ref, mag = _conv64(x64, wt.double(), b.double(), 1, 1)
    t_ref, _ = _conv64(_tf32(x64), _tf32(wt), b.double(), 1, 1)
    r1 = at["rows"][1]
    _check(out[:, r1:r1 + sizes[1][0], :sizes[1][1]].permute(0, 3, 1, 2).cpu(), ref, mag, t_ref, 2304, "view_to_view")
    engine.conv2d_f32(levels[2].to(DEV).contiguous(), hi, lo, b.to(DEV), 64, 3, stride=2,
                      out=engine.AtlasView(out, at["rows"][3], *sizes[3]))
    x64 = levels[2].permute(0, 3, 1, 2).double()
    ref, mag = _conv64(x64, wt.double(), b.double(), 2, 1)
    t_ref, _ = _conv64(_tf32(x64), _tf32(wt), b.double(), 2, 1)
    r3 = at["rows"][3]
    _check(out[:, r3:r3 + sizes[3][0], :sizes[3][1]].permute(0, 3, 1, 2).cpu(), ref, mag, t_ref, 2304, "s2_into_view")


def test_conv_f32_unsupported_combinations():
    x = torch.zeros((1, 8, 8, 48), device=DEV)
    w = torch.zeros((64, 48 * 9), device=DEV)
    with pytest.raises(RuntimeError, match="not supported"):
        engine.conv2d_f32(x, w, w, None, 64, 3)                              # cin % 32 != 0
    x = torch.zeros((1, 8, 8, 64), device=DEV)
    w = torch.zeros((64, 64), device=DEV)
    with pytest.raises(RuntimeError, match="not supported"):
        engine.conv2d_f32(x, w, w, None, 64, 1, residual=torch.zeros((1, 64, 8, 8), device=DEV), out_mode=engine.OUT_NCHW_F32)


# ---- small kernels, bit-exact ----------------------------------------------------------------------------------------
def test_pad_input_f32_exact():
    x = torch.randn((2, 37, 53, 3), generator=torch.Generator().manual_seed(1))
    got = engine.pad_input_f32(x.to(DEV)).cpu()
    want = torch.zeros((2, 43, 61, 4))
    want[:, 3:40, 3:56, :3] = x
    assert torch.equal(got, want)


def test_preprocess_u8_f32_exact():
    img = torch.randint(0, 256, (2, 100, 130, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(2))
    xp, hs, ws = engine.preprocess_u8_f32(img.to(DEV).contiguous(), 128)
    xp = xp.cpu()
    assert (hs, ws) == (128, 256)
    for i in range(2):
        want = torch.from_numpy(oracle.preprocess_u8(img[i].numpy(), 128))          # fp32 [3, hs, ws]
        assert torch.equal(xp[i, 3:3 + hs, 3:3 + ws, :3], want.permute(1, 2, 0))
    assert float(xp[:, :, :, 3].abs().max()) == 0.0


def test_resize_f32_exact():
    g = torch.Generator().manual_seed(3)
    imgs = [torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, generator=g) for h, w in ((300, 410), (97, 61))]
    xp, hs, ws, ratios = engine.preprocess_resize_u8(imgs, 160, 240, 32, f32=True)
    xp = xp.cpu()
    for i, im in enumerate(imgs):
        _, dh, dw = resize_oracle.resize_ratio(im.shape[0], im.shape[1], 160, 240)
        want = torch.zeros((3, hs, ws))
        pre = torch.from_numpy(oracle.preprocess_u8(resize_oracle.resize_bilinear(im.numpy(), dh, dw), 2))
        want[:, :pre.shape[1], :pre.shape[2]] = pre
        assert torch.equal(xp[i, 3:3 + hs, 3:3 + ws, :3], want.permute(1, 2, 0)), i


def test_maxpool_and_relu_copy_f32_exact():
    x = torch.randn((2, 33, 46, 64), generator=torch.Generator().manual_seed(4))
    got = engine.maxpool3x3s2_f32(x.to(DEV)).cpu()
    assert torch.equal(got, F.max_pool2d(x.permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1))
    atlas = torch.randn((2, 30, 20, 256), generator=torch.Generator().manual_seed(5))
    got = engine.relu_from_view_f32(engine.AtlasView(atlas.to(DEV), 8, 7, 13)).cpu()
    assert torch.equal(got, atlas[:, 8:15, :13].clamp_min(0))


# ---- model ---------------------------------------------------------------------------------------------------------------
def _rel_err(got, ref):
    return float((got - ref).abs().max() / (ref.abs().max() + 1e-12))


# Heads against fp32 references: each tensor within 5e-4 * max|ref|, and the model's worst fp32 tensor at least 4x closer
# than its worst fp16 tensor.  A per-tensor 20x bar does not hold.  The floor is this mode's own arithmetic, not the
# reference's: the fp32 oracle is within about 1.3e-6 of the same oracle run in float64, while the fp32 mode is 1e-4 -
# 2.3e-4 off.  Each split-TF32 convolution is accurate to about 1e-6 of sum|a b| per output, but the tensor cores
# accumulate in fp32 with truncation across s = 3 K / 8 MMAs (0.04 - 0.05 of single-pass TF32's error at K = 2304, see
# _check), and that error compounds through 20 - 150 layers.  On the near-constant small levels the fp16 mode reaches
# the same floor (P7 class map: 5.6e-7 fp32 against 6.5e-7 fp16), hence a per-model instead of a per-tensor ratio.


def _heads_f64(sd, backbone, x):
    """oracle/model_ref's heads (logits) in float64: its building blocks on float64 weights and input."""
    sd64 = {k: v.double() for k, v in sd.items()}
    with torch.no_grad():
        feats = model_ref.features(sd64, backbone, x.double(), False)
        return [model_ref.head(sd64, "cls_head", t) for t in feats], [model_ref.head(sd64, "box_head", t) for t in feats]


def _spread_head(sd, std=0.05, prior=0.02):
    g = torch.Generator().manual_seed(123)
    sd = dict(sd)
    sd["cls_head.8.weight"] = torch.randn(sd["cls_head.8.weight"].shape, generator=g) * std
    sd["cls_head.8.bias"] = torch.full_like(sd["cls_head.8.bias"], -float(np.log((1 - prior) / prior)))
    sd["box_head.8.weight"] = torch.randn(sd["box_head.8.weight"].shape, generator=g) * 0.02
    return sd


def _match_rate(got, ref, size, score_tol=1e-3, box_tol=1e-3):
    """As in test_gpu_model.py: the fraction of the reference detections of ONE image that have a counterpart of the same
    class within score_tol and box_tol * size pixels (rank-independent), and the worst matched deviations."""
    gs, gb, gc = got
    rs, rb, rc = ref
    n = int((rs > 0).sum())
    if n == 0:
        return 1.0, 0, (0.0, 0.0)
    scale = np.array([size] * 4 + [1.0] * (rb.shape[1] - 4), np.float32)
    hit, worst_s, worst_b = 0, 0.0, 0.0
    for i in range(n):
        db = (np.abs(gb - rb[i]) / scale).max(axis=1)
        ds = np.abs(gs - rs[i])
        cand = np.where(gc == rc[i], np.maximum(db / box_tol, ds / score_tol), np.inf)
        j = int(np.argmin(cand))
        if cand[j] <= 1.0:
            hit += 1
        if np.isfinite(cand[j]) and cand[j] < 50:
            worst_s, worst_b = max(worst_s, float(ds[j])), max(worst_b, float(db[j]))
    return hit / n, n, (worst_s, worst_b)


@pytest.mark.parametrize("backbone", ["ResNet18FPN", "ResNet50FPN"])
def test_heads_match_reference_fp32_golden(golden_dir, backbone):
    g = np.load(os.path.join(golden_dir, "model_%s.npz" % backbone))
    m = Model(backbone, classes=int(g["classes"]))
    m.load_state_dict(make_state_dict(backbone, int(g["classes"]), 9, False, int(g["seed"]))).cuda()
    x = torch.from_numpy(g["x"]).to(DEV)
    c16, b16 = m.forward_heads(x, sigmoid=True)
    c16, b16 = [t.cpu() for t in c16], [t.cpu() for t in b16]
    m.set_precision("fp32")
    cls, box = m.forward_heads(x, sigmoid=True)
    worst = [0.0, 0.0]
    for i in range(5):
        for got, h16, key in ((cls[i], c16[i], "cls%d" % i), (box[i], b16[i], "box%d" % i)):
            ref = torch.from_numpy(g[key])
            e32, e16 = _rel_err(got.cpu(), ref), _rel_err(h16, ref)
            MEASURED["golden_%s_%s" % (backbone, key)] = (e32, e16)
            assert e32 <= 5e-4, (key, e32)
            worst = [max(worst[0], e32), max(worst[1], e16)]
    MEASURED["golden_%s_worst" % backbone] = tuple(worst)
    assert worst[0] * 4 <= worst[1], worst


@pytest.mark.parametrize("backbone,shape,rotated", [("ResNet50FPN", (2, 3, 256, 384), False), ("ResNet101FPN", (1, 3, 128, 256), False),
                                                    ("ResNet34FPN", (1, 3, 128, 128), False), ("ResNet152FPN", (1, 3, 128, 128), False),
                                                    ("ResNet18FPN", (1, 3, 256, 256), True), ("ResNet50FPN", (1, 3, 160, 224), False)])
def test_heads_match_fp32_oracle(backbone, shape, rotated):
    na = 27 if rotated else 9
    sd = make_state_dict(backbone, 5, na, rotated, 3)
    x = torch.randn(shape, generator=torch.Generator().manual_seed(1))
    m = Model(backbone, classes=5, rotated_bbox=rotated).load_state_dict(sd).cuda()
    c16, b16 = [[t.cpu() for t in h] for h in m.forward_heads(x.to(DEV), sigmoid=False)]
    m.set_precision("fp32")
    cls, box = m.forward_heads(x.to(DEV), sigmoid=False)
    rc, rb = model_ref.forward_heads(sd, backbone, x, sigmoid=False)
    c64, b64 = _heads_f64(sd, backbone, x)
    worst = [0.0, 0.0, 0.0, 0.0]          # fp32 mode, fp16 mode vs the fp32 oracle; fp32 mode, fp32 oracle vs float64
    for i in range(5):
        for got, h16, ref, r64, key in ((cls[i], c16[i], rc[i], c64[i], "cls%d" % i), (box[i], b16[i], rb[i], b64[i], "box%d" % i)):
            assert tuple(got.shape) == tuple(ref.shape)
            e32, e16 = _rel_err(got.cpu(), ref), _rel_err(h16, ref)
            assert e32 <= 5e-4, (key, e32)
            worst = [max(worst[0], e32), max(worst[1], e16), max(worst[2], _rel_err(got.cpu().double(), r64)),
                     max(worst[3], _rel_err(ref.double(), r64))]
    MEASURED["oracle_%s_%s_rot%d_worst" % (backbone, "x".join(map(str, shape)), rotated)] = tuple(worst)
    assert worst[0] * 4 <= worst[1], worst
    assert worst[3] * 20 <= worst[2], worst       # the reference is not the floor


@pytest.mark.parametrize("backbone,shape", [("ResNet18FPN", (2, 3, 256, 256)), ("ResNet50FPN", (1, 3, 256, 384))])
def test_forward_end_to_end_within_1e3_of_fp32_oracle(backbone, shape):
    classes = 6
    sd = _spread_head(make_state_dict(backbone, classes, 9, False, 10))
    x = torch.randn(shape, generator=torch.Generator().manual_seed(4))
    m = Model(backbone, classes=classes).load_state_dict(sd).cuda().set_precision("fp32")
    got = [t.cpu().numpy() for t in m(x.to(DEV))]
    ref = model_ref.forward(sd, backbone, x)
    total = 0
    for img in range(shape[0]):
        rate, n, worst = _match_rate([t[img] for t in got], [t[img] for t in ref], max(shape[2:]))
        total += n
        MEASURED["e2e_%s_%d" % (backbone, img)] = (rate, n, worst)
        assert rate >= 0.99, (img, rate, n, worst)
    assert total > 20


@pytest.mark.parametrize("rotated", [False, True])
def test_full_size_800x1280_resnet50_vs_fp32_oracle(rotated):
    backbone, classes = "ResNet50FPN", 80
    na = 27 if rotated else 9
    sd = _spread_head(make_state_dict(backbone, classes, na, rotated, 21))
    x = torch.randn((1, 3, 800, 1280), generator=torch.Generator().manual_seed(6))
    m = Model(backbone, classes=classes, rotated_bbox=rotated).load_state_dict(sd).cuda().set_precision("fp32")
    assert m.fused_candidates
    got = [t.cpu().numpy()[0] for t in m(x.to(DEV))]
    ref = [t[0] for t in model_ref.forward(sd, backbone, x, rotated=rotated)]
    rate, n, worst = _match_rate(got, ref, 1280)
    MEASURED["e2e_800x1280_rot%d" % rotated] = (rate, n, worst)
    assert n > 20 and rate >= 0.95, (rate, n, worst)


# ---- behaviour -------------------------------------------------------------------------------------------------------------
def _model(seed, rotated=False, classes=6, **config):
    sd = _spread_head(make_state_dict("ResNet18FPN", classes, 27 if rotated else 9, rotated, seed))
    return Model("ResNet18FPN", classes=classes, rotated_bbox=rotated, config=config).load_state_dict(sd).cuda()


def _same(a, b):
    for u, v in zip(a, b):
        assert torch.equal(u, v)


def test_cuda_graph_replay_equals_eager_fp32():
    m = _model(10).set_precision("fp32")
    xs = [torch.randn((2, 3, 128, 256), generator=torch.Generator().manual_seed(s)).to(DEV) for s in (1, 2)]
    eager = [[t.clone() for t in m(x)] for x in xs]
    assert (eager[0][0] > 0).sum() > 5
    m.enable_cuda_graph()
    for x, e in zip(xs + xs[:1], eager + eager[:1]):
        _same(m(x), e)


@pytest.mark.parametrize("rotated", [False, True])
def test_parallel_heads_and_dense_route_fp32(rotated):
    m = _model(13, rotated).set_precision("fp32")
    x = torch.randn((2, 3, 256, 256), generator=torch.Generator().manual_seed(3)).to(DEV)
    m.parallel_heads = False
    seq = [t.clone() for t in m(x)]
    assert (seq[0] > 0).sum() > 5
    m.parallel_heads = True
    _same(m(x), seq)
    m.fused_candidates = False
    _same(m(x), seq)


def test_forward_images_and_jpeg_equal_forward_fp32():
    from PIL import Image
    m = _model(10).set_precision("fp32")
    g = torch.Generator().manual_seed(9)
    imgs = [torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, generator=g) for h, w in ((240, 320), (200, 150))]
    resize, max_size = 256, 400
    for fused in (True, False):
        m.fused_candidates = fused
        got, ratios = m.forward_images(imgs, resize, max_size)
        got = [t.clone() for t in got]
        # the batch built on the CPU: Pillow-exact resize, reference normalisation, collate -> model(x)
        pres = []
        for im in imgs:
            _, dh, dw = resize_oracle.resize_ratio(im.shape[0], im.shape[1], resize, max_size)
            pres.append(oracle.preprocess_u8(resize_oracle.resize_bilinear(im.numpy(), dh, dw), 128))
        hs, ws = max(p.shape[1] for p in pres), max(p.shape[2] for p in pres)
        x = torch.zeros((len(pres), 3, hs, ws))
        for i, p in enumerate(pres):
            x[i, :, :p.shape[1], :p.shape[2]] = torch.from_numpy(p)
        _same(got, m(x.to(DEV)))
        datas = []
        for im in imgs:
            buf = io.BytesIO()
            Image.fromarray(im.numpy()).save(buf, "JPEG", quality=90)
            datas.append(buf.getvalue())
        dec = [torch.from_numpy(np.asarray(Image.open(io.BytesIO(d)).convert("RGB")).copy()) for d in datas]
        want = [t.clone() for t in m.forward_images(dec, resize, max_size)[0]]
        jg, _, status = m.forward_jpeg(datas, resize, max_size)
        _same(jg, want)
        assert status.cpu().tolist() == [0, 0]
    m.enable_cuda_graph()
    m.fused_candidates = True
    eager = [t.clone() for t in m.forward_images(imgs, resize, max_size, canvas=(384, 512))[0]]
    m._graphs = None
    _same(eager, m.forward_images(imgs, resize, max_size, canvas=(384, 512))[0])


def test_switching_precision_round_trips():
    m = _model(15)
    x = torch.randn((1, 3, 256, 256), generator=torch.Generator().manual_seed(5)).to(DEV)
    first = [t.clone() for t in m(x)]
    h16 = [t.clone() for t in m.forward_heads(x)[0]]
    m.set_precision("fp32")
    f32 = [t.clone() for t in m(x)]
    assert not all(torch.equal(a, b) for a, b in zip(first, f32))
    m.set_precision("fp16")
    _same(m(x), first)
    _same(m.forward_heads(x)[0], h16)
    m.set_precision("fp32")
    _same(m(x), f32)
    table = m.calibrate([x], method="max")                         # calibration runs the fp16 network
    m.set_precision("int8", table)
    assert m.precision == "int8" and m._f32 is None
    q = m(x)
    assert (q[0] > 0).sum() > 0


def test_training_loss_unchanged_by_fp32():
    m = _model(16)
    x = torch.randn((2, 3, 128, 128), generator=torch.Generator().manual_seed(6)).to(DEV)
    targets = torch.tensor([[[10.0, 12.0, 40.0, 50.0, 1.0], [60.0, 20.0, 30.0, 30.0, 3.0]]] * 2, device=DEV)
    m.train()
    want = [t.clone() for t in m([x, targets])]
    m.set_precision("fp32")
    _same(m([x, targets]), want)
    m.eval()


def test_zz_report_measured():
    """Prints the measured worst cases next to each bar (pytest -s)."""
    for k, v in sorted(MEASURED.items()):
        print("fp32 measured %-40s %s" % (k, v))
