"""GPU tests of FPN training: the 1x1 / 3x3 / stride-2 weight gradient over one atlas level (odtk_conv_wgrad_ex) against
float64 on the same fp16 operands, the top-down pathway's pool-add and pyramid7's dilation bit-exact against CPU
emulation, the "fpn" scope's model gradients against CPU fp32 autograd of the oracle's FPN + heads, the reference golden,
a short SGD + GradScaler loop, and the routing / launch-count / determinism rules of the backward."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _levels(h, w):
    s = [(h // 8, w // 8), (h // 16, w // 16), (h // 32, w // 32)]
    h6, w6 = (s[2][0] - 1) // 2 + 1, (s[2][1] - 1) // 2 + 1
    return tuple(s + [(h6, w6), ((h6 - 1) // 2 + 1, (w6 - 1) // 2 + 1)])


def _geometry(n, sizes):
    """Atlas geometry of the model for five level sizes, plus each level's slice of the tile table."""
    from retinanet_examples_b200.model import Model
    at = Model("ResNet18FPN", classes=1)._atlas_for(n, tuple(sizes), torch.device(DEV))
    counts = [((h + 7) // 8) * ((w + 15) // 16) for h, w in sizes]
    starts = np.cumsum([0] + counts).tolist()
    return at, [at["tab"][starts[l]:starts[l + 1]] for l in range(5)]


def _wgrad_ex_case(n, sizes, l, x_hw, cin, ksize, stride, cout=256, seed=0):
    """g: random at level l (channels < cout), garbage at every other level; x dense.  Checks the float64 bound, the
    garbage-free result and a second call bit for bit; returns the worst ratios (w, b)."""
    from retinanet_examples_b200 import engine
    at, tabs = _geometry(n, sizes)
    gen = torch.Generator().manual_seed(seed)
    cpad = engine.pad64(cout)
    r0, (h, w) = at["rows"][l], sizes[l]
    assert (h, w) == ((x_hw[0] - 1) // stride + 1, (x_hw[1] - 1) // stride + 1)
    ha, wa = at["buf"][0].shape[1:3]
    clean = torch.zeros((n, ha, wa, cpad))
    gl = torch.randn((n, h, w, cout), generator=gen) * 0.1
    clean[:, r0:r0 + h, :w, :cout] = gl
    dirty = clean.clone()
    for k, (r, (hh, ww)) in enumerate(zip(at["rows"], sizes)):
        if k != l:
            dirty[:, r:r + hh, :ww] = torch.randn((n, hh, ww, cpad), generator=gen) * 3.0
    x = torch.randn((n, x_hw[0], x_hw[1], cin), generator=gen).half().to(DEV)
    g_clean, g_dirty = clean.half().to(DEV), dirty.half().to(DEV)
    dw, db = engine.conv_wgrad_ex(g_dirty, x, cout, ksize, stride, tabs[l], r0)
    dw2, db2 = engine.conv_wgrad_ex(g_dirty, x, cout, ksize, stride, tabs[l], r0)
    assert torch.equal(dw, dw2) and torch.equal(db, db2)                        # bit-identical run to run
    dw3, db3 = engine.conv_wgrad_ex(g_clean, x, cout, ksize, stride, tabs[l], r0)
    assert torch.equal(dw, dw3) and torch.equal(db, db3)                        # the other levels do not count
    g64 = g_clean[:, r0:r0 + h, :w, :cout].double().permute(0, 3, 1, 2)
    x64 = x.double().permute(0, 3, 1, 2)
    shape = (cout, cin, ksize, ksize)
    pad = ksize // 2
    ref = torch.nn.grad.conv2d_weight(x64, shape, g64, stride=stride, padding=pad)
    bound = torch.nn.grad.conv2d_weight(x64.abs(), shape, g64.abs(), stride=stride, padding=pad)
    u = 2.0 ** -23 * n * h * w
    r1 = float(((dw.double() - ref).abs() / (u * bound + 1e-300)).max())
    r2 = float(((db.double() - g64.sum(dim=(0, 2, 3))).abs() / (u * g64.abs().sum(dim=(0, 2, 3)) + 1e-300)).max())
    assert r1 <= 1.0 and r2 <= 1.0, (r1, r2)
    print("wgrad_ex k%d s%d n%d x%s cin %d level %d (row0 %d): worst ratio to 2^-23 s sum|gx| (w, b) = %.3g, %.3g"
          % (ksize, stride, n, x_hw, cin, l, r0, r1, r2))
    return r1, r2


@pytest.mark.parametrize("cin,l", [(128, 0), (512, 0), (1024, 1), (2048, 2)])
def test_wgrad_ex_1x1(cin, l):
    sizes = _levels(256, 384)
    _wgrad_ex_case(2, sizes, l, sizes[l], cin, 1, 1, seed=cin)


@pytest.mark.parametrize("x_hw,cin", [((25, 40), 256), ((13, 20), 512), ((7, 10), 2048), ((25, 40), 2048),
                                      ((13, 20), 256)])
def test_wgrad_ex_stride2(x_hw, cin):
    out = ((x_hw[0] - 1) // 2 + 1, (x_hw[1] - 1) // 2 + 1)
    sizes = [(32, 48), (16, 24), x_hw, out, ((out[0] - 1) // 2 + 1, (out[1] - 1) // 2 + 1)]
    _wgrad_ex_case(2, sizes, 3, x_hw, cin, 3, 2, seed=cin + x_hw[0])


@pytest.mark.parametrize("l", [0, 2])
def test_wgrad_ex_3x3_dense(l):
    sizes = _levels(256, 384)
    _wgrad_ex_case(2, sizes, l, sizes[l], 256, 3, 1, seed=l)


@pytest.mark.parametrize("size,n", [((256, 384), 1), ((256, 384), 8), ((800, 1280), 1), ((800, 1280), 8)])
def test_wgrad_ex_real_atlas_levels(size, n):
    """Every FPN layer's case at its own level of a real atlas geometry (nonzero g_row0 from level 1 on)."""
    sizes = _levels(*size)
    c5 = (size[0] // 32, size[1] // 32)
    _wgrad_ex_case(n, sizes, 1, sizes[1], 256, 3, 1, seed=1)        # smooth4
    _wgrad_ex_case(n, sizes, 2, sizes[2], 2048, 1, 1, seed=2)       # lateral5
    _wgrad_ex_case(n, sizes, 3, c5, 512, 3, 2, seed=3)              # pyramid6 (ResNet18 C5)
    _wgrad_ex_case(n, sizes, 4, sizes[3], 256, 3, 2, seed=4)        # pyramid7 over relu(P6)


# ---- the two small kernels against CPU emulation ---------------------------------------------------------------------
def _random_atlas(at, sizes, c, gen, scale=1.0):
    n, ha, wa = at["buf"][0].shape[:3]
    a = torch.zeros((n, ha, wa, c))
    for r, (h, w) in zip(at["rows"], sizes):
        a[:, r:r + h, :w] = torch.randn((n, h, w, c), generator=gen) * scale
    return a.half()


def _pool_add_emulated(a, src, dst, pool):
    """fp16_rn((float)dst + ((s00 + s01) + (s10 + s11))) in fp32 on the CPU (pixels past the src level: 0)."""
    out = a.clone()
    (sr, sh, sw), (dr, dh, dw) = src, dst
    f = torch.zeros((a.shape[0], pool * dh, pool * dw, a.shape[3]))
    hh, ww = min(sh, pool * dh), min(sw, pool * dw)
    f[:, :hh, :ww] = a[:, sr:sr + hh, :ww].float()
    if pool == 2:
        s = (f[:, 0::2, 0::2] + f[:, 0::2, 1::2]) + (f[:, 1::2, 0::2] + f[:, 1::2, 1::2])
    else:
        s = f
    out[:, dr:dr + dh, :dw] = (a[:, dr:dr + dh, :dw].float() + s).half()
    return out


@pytest.mark.parametrize("size,n", [((256, 384), 2), ((800, 1280), 1)])
def test_pool_add_bit_exact(size, n):
    from retinanet_examples_b200 import engine
    sizes = _levels(*size)
    at, _ = _geometry(n, sizes)
    gen = torch.Generator().manual_seed(n)
    a = _random_atlas(at, sizes, 256, gen, scale=100.0)
    lv = [(r, h, w) for r, (h, w) in zip(at["rows"], sizes)]
    ga = a.to(DEV)
    exp = a
    for l in range(2):                          # the FPN order: 0 -> 1, then 1 -> 2, in place
        engine.pool_add(ga, ga, lv[l], lv[l + 1], pool=2)
        exp = _pool_add_emulated(exp, lv[l], lv[l + 1], 2)
        assert torch.equal(ga.cpu(), exp), l
    other = _random_atlas(at, sizes, 256, gen).to(DEV)
    engine.pool_add(other, ga, lv[3], lv[3], pool=1)
    exp[:, lv[3][0]:lv[3][0] + lv[3][1], :lv[3][2]] = (exp[:, lv[3][0]:lv[3][0] + lv[3][1], :lv[3][2]].float()
                                                       + other.cpu()[:, lv[3][0]:lv[3][0] + lv[3][1], :lv[3][2]].float()).half()
    assert torch.equal(ga.cpu(), exp)
    # a source level that is not twice the destination: the missing pixels count as 0
    b = _random_atlas(at, sizes, 64, gen).to(DEV)
    e = _pool_add_emulated(b.cpu(), (lv[3][0], lv[3][1], lv[3][2]), (lv[4][0], lv[4][1], lv[4][2]), 2)
    engine.pool_add(b, b, lv[3], lv[4], pool=2)
    assert torch.equal(b.cpu(), e)


@pytest.mark.parametrize("size,n", [((256, 384), 2), ((800, 1280), 3)])
def test_dilate_bit_exact_and_odd_positions_stay_zero(size, n):
    from retinanet_examples_b200 import engine
    sizes = _levels(*size)
    at, _ = _geometry(n, sizes)
    gen = torch.Generator().manual_seed(5)
    dst = torch.zeros(at["buf"][0].shape, dtype=torch.float16, device=DEV)
    (r3, (h6, w6)), (r4, (h7, w7)) = (at["rows"][3], sizes[3]), (at["rows"][4], sizes[4])
    for _ in range(2):
        src = _random_atlas(at, sizes, 256, gen).to(DEV)
        engine.dilate(src, dst, (r4, h7, w7), r3)
        exp = torch.zeros(dst.shape, dtype=torch.float16)
        exp[:, r3:r3 + 2 * h7:2, 0:2 * w7:2] = src.cpu()[:, r4:r4 + h7, :w7]
        assert torch.equal(dst.cpu(), exp)
        assert 2 * (h7 - 1) <= h6 - 1 and 2 * (w7 - 1) <= w6 - 1


# ---- model level ----------------------------------------------------------------------------------------------------
def _targets(n, rotated, gen, size):
    rows = []
    H, W = size
    for i in range(n):
        t = []
        for k in range(3 + i):
            x0, y0 = float(torch.rand(1, generator=gen)) * W * 0.6, float(torch.rand(1, generator=gen)) * H * 0.6
            bw, bh = 16 + float(torch.rand(1, generator=gen)) * W * 0.35, 16 + float(torch.rand(1, generator=gen)) * H * 0.35
            c = float(torch.randint(0, 3, (1,), generator=gen))
            t.append([x0, y0, bw, bh] + ([float(torch.rand(1, generator=gen)) - 0.5] if rotated else []) + [c])
        rows.append(t)
    m = max(len(t) for t in rows)
    out = torch.full((n, m, 6 if rotated else 5), -1.0)
    for i, t in enumerate(rows):
        out[i, :len(t)] = torch.tensor(t)
    return out


def _lively(sd, seed):
    g = torch.Generator().manual_seed(seed)
    for k in sd:      # livelier heads than the init's 0.01 std, so every layer's gradient is far from zero
        if k.startswith(("cls_head", "box_head")) and k.endswith("weight"):
            sd[k] = torch.randn(sd[k].shape, generator=g) * 0.03
    return sd


def _ref_grads(m, params, st, fp16):
    """CPU fp32 autograd of oracle.model_ref._fpn + head on the model's own saved C3-C5 and its loss gradients."""
    from oracle import model_ref
    S = st["fpn"]
    cs = [S[k].permute(0, 3, 1, 2).float().cpu() for k in ("c3", "c4", "c5")]
    sd = {k: v for k, v in m._sd.items()}
    ref = {k: params[k].detach().cpu().clone().requires_grad_(True) for k in params}
    sd.update(ref)
    feats = model_ref._fpn(sd, m.backbone, *cs, fp16)
    total = 0.0
    for head in ("cls_head", "box_head"):
        for l, f in enumerate(feats):
            total = total + (model_ref.head(sd, head, f, fp16=fp16) * st["grads"][head][l].cpu()).sum()
    total.backward()
    return {k: v.grad for k, v in ref.items()}


def _errs(params, ref, scale):
    return {k: float((p.grad.cpu() / scale - ref[k]).abs().max() / ref[k].abs().max()) for k, p in params.items()}


@pytest.mark.parametrize("backbone,rotated,shape", [("ResNet18FPN", False, (2, 256, 384)), ("ResNet18FPN", True, (2, 256, 384)),
                                                    ("ResNet50FPN", False, (2, 256, 384)), ("ResNet50FPN", True, (2, 256, 384)),
                                                    ("ResNet50FPN", False, (1, 800, 1280))])
def test_model_fpn_gradients_vs_cpu_autograd(backbone, rotated, shape):
    """Every FPN weight / bias gradient against CPU fp32 autograd and against the fp16-emulating oracle, per tensor
    relative to max|ref|.  Measured on the H100: lateral3-5 and smooth3-5 at most 0.0064 (fp32) / 0.0047 (fp16-emulating),
    so their bar is 1e-2, tighter than the heads' 3e-2; pyramid6 / pyramid7 at most 0.031 / 0.019 -- at 256 x 384 P7 has
    2 x 3 pixels and P6 4 x 6, so the sum over pixels averages out little of the fp16 activations' difference -- bar 5e-2.
    The head gradients here run on the oracle's own FPN output rather than the GPU's atlas (test_gpu_train_heads.py holds
    them to 3e-2 on that): measured at most 0.038 / 0.067, bar 1e-1.  Loss scaled by 2^16, as GradScaler's initial
    scale."""
    from retinanet_examples_b200.model import Model, make_state_dict
    m = Model(backbone, classes=3, rotated_bbox=rotated)
    m.load_state_dict(_lively(make_state_dict(backbone, 3, m.num_anchors, rotated, seed=4), 11)).cuda(0)
    m.set_train_scope("fpn")
    params = dict(m.named_parameters())
    assert list(params)[:16] == m._fpn_param_names()
    m.train()
    m.want_atlas_grad = True
    g = torch.Generator().manual_seed(12)
    n, H, W = shape
    x = torch.randn((n, 3, H, W), generator=g).to(DEV)
    t = _targets(n, rotated, g, (H, W)).to(DEV)
    cls_loss, box_loss = m([x, t])
    ((cls_loss + box_loss) * 2.0 ** 16).backward()
    st = m.last_train
    e32 = _errs(params, _ref_grads(m, params, st, False), 2.0 ** 16)
    e16 = _errs(params, _ref_grads(m, params, st, True), 2.0 ** 16)
    fpn = m._fpn_param_names()
    for tag, e in (("fp32", e32), ("fp16-emulating", e16)):
        wf = max(fpn, key=e.get)
        wh = max((k for k in e if k not in fpn), key=e.get)
        print("model %s %s %s vs the %s oracle: worst FPN %s %.3g, worst head %s %.3g"
              % (backbone, "rotated" if rotated else "axis", shape, tag, wf, e[wf], wh, e[wh]))
        print("   ", {k.split(".", 2)[-1]: round(e[k], 4) for k in fpn})
    for k in params:
        bar = 1e-1 if k not in fpn else 5e-2 if ".pyramid" in k else 1e-2
        assert e32[k] < bar and e16[k] < bar, (k, e32[k], e16[k])


def test_fpn_gradients_match_the_reference_golden(golden_dir):
    """The unmodified reference's training-mode ResNet18FPN on the CPU in fp32 (oracle/gen_golden_fpn_grads.py) against
    this model on the GPU: the losses, every FPN bias gradient, the stored output channels and the per-channel gradient
    norms of every FPN weight within 3e-2 * max|ref| per tensor."""
    from oracle.gen_golden_fpn_grads import BACKBONE, CLASSES, inputs
    from retinanet_examples_b200.model import Model
    gd = np.load(os.path.join(golden_dir, "fpn_grads.npz"))
    sd, x, t = inputs()
    assert abs(float(x.double().sum()) - float(gd["x_sum"])) < 1e-6
    m = Model(BACKBONE, classes=CLASSES).load_state_dict(sd).cuda(0).set_train_scope("fpn")
    params = dict(m.named_parameters())
    m.train()
    cls_loss, box_loss = m([x.to(DEV), t.to(DEV)])
    ((cls_loss + box_loss) * 2.0 ** 16).backward()
    errs = {"cls_loss": abs(float(cls_loss) / float(gd["cls_loss"]) - 1), "box_loss": abs(float(box_loss) / float(gd["box_loss"]) - 1)}
    for name in m._fpn_param_names()[::2]:
        layer = name[:-len(".weight")]
        gw, gb = params[layer + ".weight"].grad.cpu() / 2.0 ** 16, params[layer + ".bias"].grad.cpu() / 2.0 ** 16
        ch = torch.from_numpy(gd[layer + ".channels"]).long()
        for tag, a, r in (("b", gb, gd[layer + ".bias"]), ("w", gw[ch], gd[layer + ".weight"]),
                          ("norm", gw.flatten(1).norm(dim=1), gd[layer + ".norms"])):
            r = torch.from_numpy(r)
            errs[layer + "." + tag] = float((a - r).abs().max() / r.abs().max())
    worst = max(errs, key=errs.get)
    print("golden fpn grads: worst %s %.3g; losses %.3g / %.3g" % (worst, errs[worst], errs["cls_loss"], errs["box_loss"]))
    for k, v in errs.items():
        assert v < 3e-2, (k, v)


def _cpu_loss(cls_heads, box_heads, cls_idx, box_tgt, classes):
    """The reference's _compute_loss (odtk/model.py:186-210) on class-index targets, CPU fp32 autograd."""
    cls_sum, box_sum, fg = 0.0, 0.0, 0.0
    for c, b, ci, bt in zip(cls_heads, box_heads, cls_idx, box_tgt):
        B, A = ci.shape[:2]
        c = c.view(B, A, classes, *c.shape[2:])
        target = (ci.unsqueeze(2) == torch.arange(classes).view(1, 1, -1, 1, 1)).float()
        pred = c.sigmoid()
        ce = F.binary_cross_entropy_with_logits(c, target, reduction="none")
        alpha = target * 0.25 + (1 - target) * 0.75
        pt = torch.where(target == 1, pred, 1 - pred)
        cls_sum = cls_sum + ((ci >= -1).unsqueeze(2).float() * alpha * (1 - pt) ** 2 * ce).sum()
        d = (b.view_as(bt) - bt).abs()
        l1 = torch.where(d < 0.11, 0.5 * d ** 2 / 0.11, d - 0.5 * 0.11)
        box_sum = box_sum + ((ci >= 0).unsqueeze(2).float() * l1).sum()
        fg = fg + (ci >= 0).sum().float().clamp(min=1)
    return cls_sum / fg, box_sum / fg


def test_training_loop_sgd_gradscaler_fpn_scope():
    """20 iterations of the reference's loop (SGD(lr 0.01, momentum 0.9, weight decay 1e-4), LambdaLR warm-up,
    GradScaler) in the "fpn" scope: every step's loss within 1e-2 (relative) of a CPU fp32 run of the same steps (the
    oracle's FPN + heads on the model's frozen C3-C5), the backbone stays bit-identical while the FPN weights change,
    fp16 / fp32 / INT8-network eval equal a fresh model loaded from state_dict(), and a 2^40 loss scale gives inf
    gradients: the step is skipped, nothing changes."""
    from oracle import model_ref
    from retinanet_examples_b200.model import Model, make_state_dict
    classes = 3
    sd = make_state_dict("ResNet18FPN", classes, 9, False, seed=6)
    m = Model("ResNet18FPN", classes=classes).load_state_dict(sd).cuda(0).set_train_scope("fpn")
    fpn = m._fpn_param_names()
    trainable = set(fpn) | set(m._head_param_names())
    frozen = {k: v.clone() for k, v in sd.items() if k not in trainable}
    g = torch.Generator().manual_seed(21)
    data = [(torch.randn((2, 3, 256, 384), generator=g).to(DEV), _targets(2, False, g, (256, 384)).to(DEV)) for _ in range(2)]
    opt = torch.optim.SGD(m.parameters(), lr=0.01, weight_decay=1e-4, momentum=0.9)
    sched = lambda it: 0.9 * it / 1000 + 0.1 if it <= 1000 else 1.0       # noqa: E731  (odtk/train.py:62-65)
    scheduler = torch.optim.lr_scheduler.LambdaLR(opt, sched)
    scaler = torch.amp.GradScaler("cuda")
    ref_p = {k: p.detach().cpu().clone().requires_grad_(True) for k, p in m.named_parameters()}
    ref_sd = dict(m._sd)
    ref_sd.update(ref_p)
    ref_opt = torch.optim.SGD(list(ref_p.values()), lr=0.01, weight_decay=1e-4, momentum=0.9)
    ref_sched = torch.optim.lr_scheduler.LambdaLR(ref_opt, sched)
    m.want_atlas_grad = True                                                     # keeps last_train: C3-C5
    m.train()
    losses, ref_losses, cache = [], [], {}
    for it in range(20):
        x, t = data[it % 2]
        opt.zero_grad()
        cls_loss, box_loss = m([x, t])
        if it % 2 not in cache:
            S, views = m.last_train["fpn"], m.last_train["views"]
            cs = [S[k].permute(0, 3, 1, 2).float().cpu() for k in ("c3", "c4", "c5")]
            tg = [m._extract_targets(t, x.shape[-1] // v.w, (v.h, v.w)) for v in views]
            cache[it % 2] = (cs, [a.cpu() for a, _, _ in tg], [b.cpu() for _, b, _ in tg])
        scaler.scale(cls_loss + box_loss).backward()
        before = scaler.get_scale()
        scaler.step(opt)
        scaler.update()
        skipped = scaler.get_scale() < before
        scheduler.step()
        losses.append(float((cls_loss + box_loss).detach()))
        cs, ci, bt = cache[it % 2]
        ref_opt.zero_grad()
        feats = model_ref._fpn(ref_sd, "ResNet18FPN", *cs, False)
        rc, rb = _cpu_loss([model_ref.head(ref_sd, "cls_head", f) for f in feats],
                           [model_ref.head(ref_sd, "box_head", f) for f in feats], ci, bt, classes)
        (rc + rb).backward()
        if not skipped:
            ref_opt.step()
        ref_sched.step()
        ref_losses.append(float((rc + rb).detach()))
    dev = max(abs(a - b) / b for a, b in zip(losses, ref_losses))
    print("fpn scope losses", [round(v, 4) for v in losses])
    print("cpu fp32 losses", [round(v, 4) for v in ref_losses], "worst relative difference %.3g" % dev)
    assert all(math.isfinite(v) for v in losses)
    assert dev < 1e-2, dev
    m.want_atlas_grad = False
    trained = m.state_dict()
    for k, v in frozen.items():
        assert torch.equal(trained[k], v), k
    for k in fpn[::2]:
        assert not torch.equal(trained[k], sd[k]), k
    m.eval()
    x = data[0][0]
    fresh = Model("ResNet18FPN", classes=classes).load_state_dict({k: v.clone() for k, v in trained.items()}).cuda(0)
    for a, b in zip(m(x), fresh(x)):
        assert torch.equal(a, b)
    m.set_precision("fp32")
    fresh.set_precision("fp32")
    for a, b in zip(m(x), fresh(x)):
        assert torch.equal(a, b)
    table = fresh.calibrate([x.cpu()], scope="network")
    m.set_precision("int8", table, scope="network")
    fresh.set_precision("int8", table, scope="network")
    for a, b in zip(m(x), fresh(x)):
        assert torch.equal(a, b)
    m.set_precision("fp16")
    # absurd scale: inf gradients, the step is skipped and the parameters stay as they are
    m.train()
    before = {k: p.detach().clone() for k, p in m.named_parameters()}
    big = torch.amp.GradScaler("cuda", init_scale=2.0 ** 40)
    opt.zero_grad()
    cls_loss, box_loss = m(list(data[0]))
    big.scale(cls_loss + box_loss).backward()
    assert any(not bool(torch.isfinite(p.grad).all()) for p in m.parameters() if p.grad is not None)
    big.step(opt)
    big.update()
    assert big.get_scale() < 2.0 ** 40
    for k, p in m.named_parameters():
        assert torch.equal(p.detach(), before[k]), k


def _model(scope="fpn", seed=6):
    from retinanet_examples_b200.model import Model, make_state_dict
    sd = _lively(make_state_dict("ResNet18FPN", 3, 9, False, seed=seed), seed)
    m = Model("ResNet18FPN", classes=3).load_state_dict(sd).cuda(0).set_train_scope(scope)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((2, 3, 256, 384), generator=g).to(DEV)
    t = _targets(2, False, g, (256, 384)).to(DEV)
    return m, x, t


def _step(m, x, t):
    """One forward + backward; returns the launches of the backward."""
    from retinanet_examples_b200 import engine
    m.zero_grad()
    m.train()
    cls_loss, box_loss = m([x, t])
    n0 = engine.STATS["launches"]
    ((cls_loss + box_loss) * 1024.0).backward()
    torch.cuda.synchronize()
    return engine.STATS["launches"] - n0


def test_frozen_fpn_layers_and_determinism():
    """requires_grad=False on single FPN layers: no .grad there, every other gradient unchanged; two backward passes
    give bit-identical .grad."""
    m, x, t = _model()
    params = dict(m.named_parameters())
    _step(m, x, t)
    ref = {k: p.grad.clone() for k, p in params.items()}
    assert all(int(g.count_nonzero()) > 0 for g in ref.values())
    _step(m, x, t)
    for k, p in params.items():
        assert torch.equal(p.grad, ref[k]), k                                   # deterministic
    pre = "backbones.ResNet18FPN."
    for frozen in (["smooth4.weight", "smooth4.bias"], ["pyramid6.weight"], ["lateral5.weight", "lateral5.bias"],
                   ["pyramid7.weight", "pyramid7.bias", "lateral3.bias"]):
        for k in frozen:
            params[pre + k].requires_grad_(False)
        _step(m, x, t)
        for k, p in params.items():
            if k[len(pre):] in frozen:
                assert p.grad is None, k
            else:
                assert torch.equal(p.grad, ref[k]), (frozen, k)
        for k in frozen:
            params[pre + k].requires_grad_(True)


def test_all_fpn_frozen_equals_the_heads_scope():
    """With every FPN parameter frozen in the "fpn" scope, the head gradients equal those of the "heads" scope bit for
    bit, with as many launches per backward."""
    mh, x, t = _model("heads")
    heads = dict(mh.named_parameters())
    nh = _step(mh, x, t)
    mf, _, _ = _model("fpn")
    pf = dict(mf.named_parameters())
    for k in mf._fpn_param_names():
        pf[k].requires_grad_(False)
    nf = _step(mf, x, t)
    assert nf == nh, (nf, nh)
    for k, p in heads.items():
        assert torch.equal(pf[k].grad, p.grad), k
    for k in mf._fpn_param_names():
        assert pf[k].grad is None
    # and the default scope lists exactly the head parameters, with their identity kept across scope changes
    assert list(dict(mf.set_train_scope("heads").named_parameters())) == list(heads)
    assert all(p is pf[k] for k, p in mf.named_parameters())
