"""GPU tests of head training: the weight-gradient kernel (odtk_conv_wgrad) and the masked input gradient
(odtk_conv2d_dgrad) against float64 on the same fp16 operands, the gradient atlas (odtk_grad_to_atlas), the model-level
head gradients against CPU fp32 autograd of the oracle's heads, and a short SGD + GradScaler training loop."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _levels(h, w):
    """Image size -> the five pyramid level sizes of the ResNet FPNs (P3 = /8 ... P7; 800 x 1280 has odd P6 / P7)."""
    s = [(h // 8, w // 8), (h // 16, w // 16), (h // 32, w // 32)]
    h6, w6 = (s[2][0] - 1) // 2 + 1, (s[2][1] - 1) // 2 + 1
    return tuple(s + [(h6, w6), ((h6 - 1) // 2 + 1, (w6 - 1) // 2 + 1)])


def _atlas_geometry(n, h, w):
    from retinanet_examples_b200.model import Model
    m = Model("ResNet18FPN", classes=1)
    return m._atlas_for(n, _levels(h, w), torch.device(DEV))


def _fill(at, sizes, c, gen, relu=False, cvalid=None, scale=1.0):
    """fp16 atlas [n, rows, width, c] on the GPU, random at the levels' pixels (channels < cvalid), zero elsewhere."""
    n, ha, wa = at["buf"][0].shape[:3]
    a = torch.zeros((n, ha, wa, c), dtype=torch.float32)
    cv = c if cvalid is None else cvalid
    for r, (h, w) in zip(at["rows"], sizes):
        v = torch.randn((n, h, w, cv), generator=gen) * scale
        a[:, r:r + h, :w, :cv] = F.relu(v) if relu else v
    return a.half().to(DEV)


def _dense_levels(a, at, sizes):
    """[n, c, h, w] float64 views of every level (CPU)."""
    a = a.double().cpu()
    return [a[:, r:r + h, :w, :].permute(0, 3, 1, 2).contiguous() for r, (h, w) in zip(at["rows"], sizes)]


def _wgrad_ref(gs, xs, cout, cin):
    dw = torch.zeros((cout, cin, 3, 3), dtype=torch.float64, device=DEV)
    bound = torch.zeros_like(dw)
    db = torch.zeros(cout, dtype=torch.float64, device=DEV)
    dbb = torch.zeros_like(db)
    for g, x in zip(gs, xs):
        g, x = g[:, :cout].to(DEV), x.to(DEV)
        dw += torch.nn.grad.conv2d_weight(x, dw.shape, g, padding=1)
        bound += torch.nn.grad.conv2d_weight(x.abs(), dw.shape, g.abs(), padding=1)
        db += g.sum(dim=(0, 2, 3))
        dbb += g.abs().sum(dim=(0, 2, 3))
    return dw, bound, db, dbb


WGRAD_RATIOS = {}


def _check_wgrad(dw, db, ref, s):
    rdw, bound, rdb, dbb = ref
    u = 2.0 ** -23 * s
    r1 = float(((dw.double() - rdw).abs() / (u * bound + 1e-300)).max())
    r2 = float(((db.double() - rdb).abs() / (u * dbb + 1e-300)).max())
    assert r1 <= 1.0 and r2 <= 1.0, (r1, r2)
    return r1, r2


@pytest.mark.parametrize("size,n,cout", [((256, 384), 1, 256), ((256, 384), 8, 256), ((256, 384), 2, 720),
                                         ((256, 384), 2, 36), ((256, 384), 2, 54), ((800, 1280), 1, 256),
                                         ((800, 1280), 8, 256), ((800, 1280), 1, 720)])
def test_wgrad_atlas_vs_float64(size, n, cout):
    from retinanet_examples_b200 import engine
    sizes = _levels(*size)
    at = _atlas_geometry(n, *size)
    gen = torch.Generator().manual_seed(cout + n)
    cpad = engine.pad64(cout)
    g = _fill(at, sizes, cpad, gen, cvalid=cout, scale=0.1)
    x = _fill(at, sizes, 256, gen, relu=True)
    dw, db = engine.conv_wgrad(g, x, cout, tile_tab=at["tab"])
    dw2, db2 = engine.conv_wgrad(g, x, cout, tile_tab=at["tab"])
    assert torch.equal(dw, dw2) and torch.equal(db, db2)                      # bit-identical run to run
    s = n * sum(h * w for h, w in sizes)
    ref = _wgrad_ref(_dense_levels(g, at, sizes), _dense_levels(x, at, sizes), cout, 256)
    WGRAD_RATIOS[(size, n, cout)] = _check_wgrad(dw, db, ref, s)
    print("wgrad", size, n, cout, "worst ratio to 2^-23 s sum|gx| (w, b):", WGRAD_RATIOS[(size, n, cout)])


@pytest.mark.parametrize("n,h,w,cout", [(2, 20, 36, 256), (1, 13, 7, 64), (3, 33, 50, 128)])
def test_wgrad_dense_vs_float64(n, h, w, cout):
    from retinanet_examples_b200 import engine
    gen = torch.Generator().manual_seed(h * w)
    g = (torch.randn((n, h, w, cout), generator=gen) * 0.1).half().to(DEV)
    x = torch.randn((n, h, w, 256), generator=gen).half().to(DEV)
    dw, db = engine.conv_wgrad(g, x, cout)
    ref = _wgrad_ref([g.double().permute(0, 3, 1, 2)], [x.double().permute(0, 3, 1, 2)], cout, 256)
    print("wgrad dense", (n, h, w, cout), _check_wgrad(dw, db, ref, n * h * w))


def _dgrad_ref(g, wt, cin):
    """d/dx of conv2d(x, wt, padding=1) for output gradient g (float64, NCHW)."""
    x = torch.zeros((g.shape[0], cin, g.shape[2], g.shape[3]), dtype=torch.float64, device=DEV, requires_grad=True)
    gx, = torch.autograd.grad(F.conv2d(x, wt, padding=1), x, g)
    xa = torch.zeros_like(x, requires_grad=True)
    bx, = torch.autograd.grad(F.conv2d(xa, wt.abs(), padding=1), xa, g.abs())
    return gx, bx


@pytest.mark.parametrize("size,n,cout", [((256, 384), 2, 256), ((256, 384), 1, 720), ((800, 1280), 2, 36),
                                         ((800, 1280), 1, 256)])
def test_masked_dgrad_vs_float64(size, n, cout):
    """Masked input gradient over the atlas, and d(atlas) as the sum of two towers' input gradients (residual addend):
    within the fp16 output rounding plus 2^-23 * K * sum|g w|; gap rows and columns right of the narrow levels stay 0."""
    from retinanet_examples_b200 import engine
    sizes = _levels(*size)
    at = _atlas_geometry(n, *size)
    gen = torch.Generator().manual_seed(7 * cout + n)
    cpad = engine.pad64(cout)
    g1 = _fill(at, sizes, cpad, gen, cvalid=cout, scale=0.1)
    g2 = _fill(at, sizes, cpad, gen, cvalid=cout, scale=0.1)
    mask = _fill(at, sizes, 256, gen, relu=True)
    w1 = (torch.randn((cout, 256, 3, 3), generator=gen) * 0.02).half().float().to(DEV)
    w2 = (torch.randn((cout, 256, 3, 3), generator=gen) * 0.02).half().float().to(DEV)
    out1 = engine.conv2d_dgrad(g1, engine.pack_weight_dgrad(w1, cpad), 256, mask=mask, tile_tab=at["tab"])
    a1 = engine.conv2d_dgrad(g1, engine.pack_weight_dgrad(w1, cpad), 256, tile_tab=at["tab"])
    a12 = engine.conv2d_dgrad(g2, engine.pack_weight_dgrad(w2, cpad), 256, residual=a1, tile_tab=at["tab"])
    valid = torch.zeros(out1.shape[1:3], dtype=torch.bool)
    for r, (h, w) in zip(at["rows"], sizes):
        valid[r:r + h, :w] = True
    for t in (out1, a1, a12):
        assert int(t[:, ~valid.to(DEV)].count_nonzero()) == 0
    K = 9 * cpad
    gl1, gl2 = _dense_levels(g1, at, sizes), _dense_levels(g2, at, sizes)
    ml, o1, oa1, oa12 = (_dense_levels(t, at, sizes) for t in (mask, out1, a1, a12))
    worst = 0.0
    for l in range(5):
        r1, b1 = _dgrad_ref(gl1[l][:, :cout].to(DEV), w1.double(), 256)
        r2, b2 = _dgrad_ref(gl2[l][:, :cout].to(DEV), w2.double(), 256)
        m = ml[l].to(DEV) > 0
        for got, ref, bnd in ((o1[l].to(DEV), torch.where(m, r1, torch.zeros_like(r1)), b1),
                              (oa1[l].to(DEV), r1, b1),
                              (oa12[l].to(DEV), oa1[l].to(DEV) + r2, b2)):
            tol = 2.0 ** -11 * ref.abs() + 2.0 ** -23 * K * bnd + 2.0 ** -24
            ratio = float(((got - ref).abs() / tol).max())
            worst = max(worst, ratio)
            assert ratio <= 1.0, (l, ratio)
        assert bool((o1[l].to(DEV)[~m] == 0).all())
    print("dgrad", size, n, cout, "worst ratio", worst)


def test_grad_to_atlas_scale_pad_and_overflow():
    from retinanet_examples_b200 import engine
    sizes = _levels(256, 384)
    at = _atlas_geometry(2, 256, 384)
    gen = torch.Generator().manual_seed(3)
    grads = [torch.randn((2, 54, h, w), generator=gen).to(DEV) for h, w in sizes]
    grads[1][0, 5, 3, 4] = 1e30                                               # overflows fp16 after scaling
    atlas = torch.zeros(at["buf"][0].shape[:3] + (64,), dtype=torch.float16, device=DEV)
    engine.grad_to_atlas(grads, at["rows"], 4.0, atlas)
    for l, ((h, w), r) in enumerate(zip(sizes, at["rows"])):
        lv = atlas[:, r:r + h, :w]
        exp = (grads[l] * 4.0).permute(0, 2, 3, 1).half()
        assert torch.equal(lv[..., :54], exp)
        assert int(lv[..., 54:].count_nonzero()) == 0
    assert torch.isinf(atlas[0, at["rows"][1] + 3, 4, 5]) and float(atlas[0, at["rows"][1] + 3, 4, 5]) > 0
    valid = torch.zeros(atlas.shape[1:3], dtype=torch.bool)
    for r, (h, w) in zip(at["rows"], sizes):
        valid[r:r + h, :w] = True
    assert int(atlas[:, ~valid.to(DEV)].count_nonzero()) == 0


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
    w = 6 if rotated else 5
    out = torch.full((n, m, w), -1.0)
    for i, t in enumerate(rows):
        out[i, :len(t)] = torch.tensor(t)
    return out


@pytest.mark.parametrize("backbone,rotated", [("ResNet18FPN", False), ("ResNet18FPN", True), ("ResNet50FPN", False),
                                              ("ResNet50FPN", True)])
def test_model_head_gradients_vs_cpu_autograd(backbone, rotated):
    """The GPU model's own fp16 atlas and GPU loss gradients through CPU fp32 autograd of oracle.model_ref.head: every
    head weight / bias gradient within 3e-2 * max|ref| per tensor (fp16 activations and weights against fp32, the
    forward's fp32-oracle bar), d(atlas) within 1e-1: it is per pixel, with no sum over pixels to average out the fp16
    forward's activation differences and the ReLU masks they flip (measured on the H100: 0.048 - 0.092; parameters 0.010 - 0.027).  The loss
    is scaled by 2^16 as GradScaler's initial scale does: unscaled head gradients sit in fp16's subnormal range."""
    from oracle import model_ref
    from retinanet_examples_b200.model import Model, make_state_dict
    classes = 3
    m = Model(backbone, classes=classes, rotated_bbox=rotated)
    sd = make_state_dict(backbone, classes, m.num_anchors, rotated, seed=4)
    g = torch.Generator().manual_seed(11)
    for k in sd:      # livelier heads than the init's 0.01 std, so every layer's gradient is far from zero
        if k.startswith(("cls_head", "box_head")) and k.endswith("weight"):
            sd[k] = torch.randn(sd[k].shape, generator=g) * 0.03
    m.load_state_dict(sd).cuda(0)
    params = dict(m.named_parameters())
    m.train()
    m.want_atlas_grad = True
    x = torch.randn((2, 3, 256, 384), generator=g).to(DEV)
    t = _targets(2, rotated, g, (256, 384)).to(DEV)
    cls_loss, box_loss = m([x, t])
    ((cls_loss + box_loss) * 2.0 ** 16).backward()
    st = m.last_train
    at = st["at"]
    sizes = [(v.h, v.w) for v in st["views"]]
    feats = [v.dense().permute(0, 3, 1, 2).float().cpu().requires_grad_(True) for v in st["views"]]
    ref_sd = {k: params[k].detach().cpu().clone().requires_grad_(True) for k in params}
    total = 0.0
    for head in ("cls_head", "box_head"):
        for l, f in enumerate(feats):
            out = model_ref.head(ref_sd, head, f)
            total = total + (out * st["grads"][head][l].cpu()).sum()
    total.backward()
    # the fp16-emulating oracle (weights and tower activations rounded to fp16 where the GPU stores them, so the same ReLU
    # masks): measured 0.039 - 0.045 on the H100, no closer than the fp32 oracle -- the difference left is the fp16
    # storage of the gradients between layers, not the activations
    f16 = [f.detach().clone().requires_grad_(True) for f in feats]
    sd16 = {k: params[k].detach().cpu().clone().requires_grad_(True) for k in params}
    total16 = 0.0
    for head in ("cls_head", "box_head"):
        for l, f in enumerate(f16):
            total16 = total16 + (model_ref.head(sd16, head, f, fp16=True) * st["grads"][head][l].cpu()).sum()
    total16.backward()
    w16 = 0.0
    for k, p in params.items():
        ref = sd16[k].grad
        w16 = max(w16, float((p.grad.cpu() / 2.0 ** 16 - ref).abs().max() / ref.abs().max()))
    for l, ((h, w), r) in enumerate(zip(sizes, at["rows"])):
        got = m.last_atlas_grad[:, r:r + h, :w].permute(0, 3, 1, 2).float().cpu() / 2.0 ** 16
        w16 = max(w16, float((got - f16[l].grad).abs().max() / f16[l].grad.abs().max()))
    print("model", backbone, "rotated" if rotated else "axis", "vs the fp16-emulating oracle: worst %.3g" % w16)
    assert w16 < 6e-2, w16
    worst = {}
    for k, p in params.items():
        ref = ref_sd[k].grad
        err = float((p.grad.cpu() / 2.0 ** 16 - ref).abs().max() / ref.abs().max())
        worst[k] = err
        assert err < 3e-2, (k, err)
    da = m.last_atlas_grad
    for l, ((h, w), r) in enumerate(zip(sizes, at["rows"])):
        ref = feats[l].grad
        got = da[:, r:r + h, :w].permute(0, 3, 1, 2).float().cpu() / 2.0 ** 16
        err = float((got - ref).abs().max() / ref.abs().max())
        worst["atlas%d" % l] = err
        assert err < 1e-1, ("atlas", l, err)
    wp = max(v for k, v in worst.items() if not k.startswith("atlas"))
    wa = max(v for k, v in worst.items() if k.startswith("atlas"))
    print("model", backbone, "rotated" if rotated else "axis", "worst err / max|ref|: params %.3g, atlas %.3g" % (wp, wa))


def test_training_loop_sgd_gradscaler():
    """The first 20 iterations of the reference's loop (odtk/train.py: SGD(lr 0.01, momentum 0.9, weight decay 1e-4), its
    LambdaLR warm-up over the default 1000 iterations, GradScaler) on a fixed synthetic set: every step's loss within 1e-2
    (relative) of a CPU fp32 run of the same steps,
    the loss falls, backbone / FPN weights stay bit-identical, eval detections equal those of a fresh model loaded from
    the trained state_dict, and an absurd loss scale (2^40) gives inf gradients: the step is skipped, nothing changes."""
    from retinanet_examples_b200.model import Model, make_state_dict
    classes = 3
    sd = make_state_dict("ResNet18FPN", classes, 9, False, seed=6)
    m = Model("ResNet18FPN", classes=classes).load_state_dict(sd).cuda(0)
    frozen = {k: v.clone() for k, v in sd.items() if not k.startswith(("cls_head", "box_head"))}
    g = torch.Generator().manual_seed(21)
    data = [(torch.randn((2, 3, 256, 384), generator=g).to(DEV), _targets(2, False, g, (256, 384)).to(DEV)) for _ in range(2)]
    opt = torch.optim.SGD(m.parameters(), lr=0.01, weight_decay=1e-4, momentum=0.9)
    sched = lambda it: 0.9 * it / 1000 + 0.1 if it <= 1000 else 1.0       # noqa: E731  (odtk/train.py:62-65)
    scheduler = torch.optim.lr_scheduler.LambdaLR(opt, sched)
    scaler = torch.amp.GradScaler("cuda")
    # CPU fp32 run of the same steps: the oracle's heads (model_ref.head) on the same frozen fp16 features and targets, the
    # reference's loss, the same SGD / LambdaLR, and the steps GradScaler skipped on the GPU skipped too
    from oracle import model_ref
    ref_sd = {k: p.detach().cpu().clone().requires_grad_(True) for k, p in m.named_parameters()}
    ref_opt = torch.optim.SGD(list(ref_sd.values()), lr=0.01, weight_decay=1e-4, momentum=0.9)
    ref_sched = torch.optim.lr_scheduler.LambdaLR(ref_opt, sched)
    m.want_atlas_grad = True                                                     # keeps last_train: the features
    m.train()
    losses, ref_losses, cache = [], [], {}
    for it in range(20):
        x, t = data[it % 2]
        opt.zero_grad()
        cls_loss, box_loss = m([x, t])
        if it % 2 not in cache:
            views = m.last_train["views"]
            feats = [v.dense().permute(0, 3, 1, 2).float().cpu() for v in views]
            tg = [m._extract_targets(t, x.shape[-1] // v.w, (v.h, v.w)) for v in views]
            cache[it % 2] = (feats, [a.cpu() for a, _, _ in tg], [b.cpu() for _, b, _ in tg])
        scaler.scale(cls_loss + box_loss).backward()
        before = scaler.get_scale()
        scaler.step(opt)
        scaler.update()
        skipped = scaler.get_scale() < before
        scheduler.step()
        losses.append(float((cls_loss + box_loss).detach()))
        feats, ci, bt = cache[it % 2]
        ref_opt.zero_grad()
        rc, rb = _cpu_loss([model_ref.head(ref_sd, "cls_head", f) for f in feats],
                           [model_ref.head(ref_sd, "box_head", f) for f in feats], ci, bt, classes)
        (rc + rb).backward()
        if not skipped:
            ref_opt.step()
        ref_sched.step()
        ref_losses.append(float((rc + rb).detach()))
    dev = max(abs(a - b) / b for a, b in zip(losses, ref_losses))
    print("losses", [round(v, 4) for v in losses])
    print("cpu fp32 losses", [round(v, 4) for v in ref_losses], "worst relative difference %.3g" % dev)
    assert all(math.isfinite(v) for v in losses)
    assert sum(losses[-4:]) < 0.95 * sum(losses[:4]), losses
    assert dev < 1e-2, dev
    m.want_atlas_grad = False
    trained = m.state_dict()
    for k, v in frozen.items():
        assert torch.equal(trained[k], v), k
    assert not torch.equal(trained["cls_head.0.weight"], sd["cls_head.0.weight"])
    m.eval()
    x = data[0][0]
    got = m(x)
    fresh = Model("ResNet18FPN", classes=classes).load_state_dict({k: v.clone() for k, v in trained.items()}).cuda(0)
    exp = fresh(x)
    for a, b in zip(got, exp):
        assert torch.equal(a, b)
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


def _trained_model(classes=3, seed=6):
    from retinanet_examples_b200.model import Model, make_state_dict
    sd = make_state_dict("ResNet18FPN", classes, 9, False, seed=seed)
    m = Model("ResNet18FPN", classes=classes).load_state_dict(sd).cuda(0)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((2, 3, 256, 384), generator=g).to(DEV)
    t = _targets(2, False, g, (256, 384)).to(DEV)
    return m, x, t


def test_fp32_and_fp16_eval_use_the_stepped_weights():
    """After an SGD step, eval forwards in fp16 and in fp32 equal those of a fresh model loaded from state_dict()."""
    from retinanet_examples_b200.model import Model
    m, x, t = _trained_model()
    m.set_precision("fp32")
    m.eval()
    m(x)                                           # packs the fp32 weights before training
    opt = torch.optim.SGD(m.parameters(), lr=0.01, momentum=0.9)
    m.train()
    cls_loss, box_loss = m([x, t])
    ((cls_loss + box_loss) * 1024.0).backward()
    opt.step()
    m.eval()
    got32 = m(x)
    fresh = Model("ResNet18FPN", classes=3).load_state_dict({k: v.clone() for k, v in m.state_dict().items()}).cuda(0)
    fresh.set_precision("fp32")
    for a, b in zip(got32, fresh(x)):
        assert torch.equal(a, b)
    m.set_precision("fp16")
    fresh.set_precision("fp16")
    for a, b in zip(m(x), fresh(x)):
        assert torch.equal(a, b)


def test_gradient_routing_and_frozen_parameters():
    """d cls_loss reaches only cls_head.*, d box_loss only box_head.*; a parameter with requires_grad=False gets no .grad
    while the layers below it still get theirs (equal to a run where it is trainable); box-head-only training with
    want_atlas_grad still gives d(atlas) its box-tower share."""
    m, x, t = _trained_model()
    params = dict(m.named_parameters())
    m.train()
    cls_loss, _ = m([x, t])
    (cls_loss * 1024.0).backward()
    for k, p in params.items():
        assert (p.grad is None) == k.startswith("box_head"), k
    m.zero_grad()
    _, box_loss = m([x, t])
    (box_loss * 1024.0).backward()
    for k, p in params.items():
        assert (p.grad is None) == k.startswith("cls_head"), k
    ref = {k: p.grad.clone() for k, p in params.items() if p.grad is not None}
    m.zero_grad()
    params["box_head.4.weight"].requires_grad_(False)
    params["box_head.4.bias"].requires_grad_(False)
    _, box_loss = m([x, t])
    (box_loss * 1024.0).backward()
    assert params["box_head.4.weight"].grad is None and params["box_head.4.bias"].grad is None
    for k in ("box_head.0.weight", "box_head.0.bias", "box_head.2.weight", "box_head.6.weight", "box_head.8.weight"):
        assert torch.equal(params[k].grad, ref[k]), k
    m.zero_grad()
    for k, p in params.items():
        p.requires_grad_(k.startswith("box_head"))
    m.want_atlas_grad = True
    cls_loss, box_loss = m([x, t])
    ((cls_loss + box_loss) * 1024.0).backward()
    assert all(p.grad is None for k, p in params.items() if k.startswith("cls_head"))
    assert m.last_atlas_grad is not None and int(m.last_atlas_grad.count_nonzero()) > 0


def test_head_gradients_match_the_reference_golden(golden_dir):
    """The unmodified reference's training-mode ResNet18FPN on the CPU in fp32 (FixedBatchNorm, oracle/
    gen_golden_head_grads.py) against this model on the GPU (fp16 through the whole network, loss scaled by 2^16): the
    losses, the full gradients of both final layers, every bias gradient, the stored tower channels and the per-channel
    gradient norms of every tower layer within 3e-2 * max|ref| per tensor."""
    import os

    import numpy as np
    from oracle.gen_golden_head_grads import BACKBONE, CLASSES, inputs
    from retinanet_examples_b200.model import Model
    gd = np.load(os.path.join(golden_dir, "head_grads.npz"))
    sd, x, t = inputs()
    assert abs(float(x.double().sum()) - float(gd["x_sum"])) < 1e-6
    m = Model(BACKBONE, classes=CLASSES).load_state_dict(sd).cuda(0)
    params = dict(m.named_parameters())
    m.train()
    cls_loss, box_loss = m([x.to(DEV), t.to(DEV)])
    ((cls_loss + box_loss) * 2.0 ** 16).backward()
    errs = {"cls_loss": abs(float(cls_loss) / float(gd["cls_loss"]) - 1), "box_loss": abs(float(box_loss) / float(gd["box_loss"]) - 1)}
    for head in ("cls_head", "box_head"):
        for i in (0, 2, 4, 6, 8):
            name = "%s.%d" % (head, i)
            gw, gb = params[name + ".weight"].grad.cpu() / 2.0 ** 16, params[name + ".bias"].grad.cpu() / 2.0 ** 16
            pairs = [("b", gb, torch.from_numpy(gd[name + ".bias"]))]
            if i == 8:
                pairs.append(("w", gw, torch.from_numpy(gd[name + ".weight"])))
            else:
                ch = torch.from_numpy(gd[name + ".channels"]).long()
                pairs.append(("w", gw[ch], torch.from_numpy(gd[name + ".weight"])))
                pairs.append(("norm", gw.flatten(1).norm(dim=1), torch.from_numpy(gd[name + ".norms"])))
            for tag, a, r in pairs:
                errs[name + "." + tag] = float((a - r).abs().max() / r.abs().max())
    worst = max(errs, key=errs.get)
    print("golden head grads: worst %s %.3g; losses %.3g / %.3g" % (worst, errs[worst], errs["cls_loss"], errs["box_loss"]))
    for k, v in errs.items():
        assert v < 3e-2, (k, v)


def _cpu_loss(cls_heads, box_heads, cls_idx, box_tgt, classes):
    """The reference's _compute_loss (odtk/model.py:186-210, FocalLoss / SmoothL1Loss of odtk/loss.py) on class-index
    targets, CPU fp32 autograd."""
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
