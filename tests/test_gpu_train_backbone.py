"""GPU tests of training ResNet stages 3-4 (scopes "layer4" / "layer3"): the dense-G, 1x1 stride-2 and BatchNorm-scaled
weight gradient (odtk_conv_wgrad_ex) and the masked 1x1 input gradient (odtk_conv2d_dgrad) against float64 on the same
fp16 operands, the atlas-level -> dense copy and stride-2 scatter (odtk_dilate_ex_f16) bit-exact, every layer3 / layer4
weight gradient of the model against CPU autograd of the oracle's blocks + FPN + heads, the reference golden, parameter
order and identity, scope equivalences and a short SGD + GradScaler loop."""
import math
import os

import numpy as np
import pytest
import torch

from test_gpu_train_fpn import _cpu_loss, _lively, _targets

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _rnd(gen, *shape, scale=1.0):
    return (torch.randn(shape, generator=gen) * scale).half()


@pytest.mark.parametrize("n,h,w,cin,cout,ksize,stride", [
    (2, 16, 24, 1024, 2048, 1, 2), (1, 13, 21, 1024, 2048, 1, 2), (2, 13, 21, 128, 256, 1, 2),   # downsamples, odd sizes
    (2, 8, 12, 2048, 512, 1, 1), (1, 25, 40, 512, 512, 3, 1), (2, 17, 23, 256, 256, 3, 2)])     # dense G, up to 2048
def test_dense_wgrad_with_bn_scale_vs_float64(n, h, w, cin, cout, ksize, stride):
    """dW * row_scale against float64 conv2d_weight on the same fp16 operands (relative to sum |g x| per weight, the
    fp32-accumulation bound), bit-identical on a rerun, and the unscaled result times the scale."""
    from retinanet_examples_b200 import engine
    gen = torch.Generator().manual_seed(n * h * w + cin + ksize)
    oh, ow = (h - 1) // stride + 1, (w - 1) // stride + 1
    x, g = _rnd(gen, n, h, w, cin), _rnd(gen, n, oh, ow, cout, scale=0.1)
    scale = torch.rand(cout, generator=gen) + 0.5
    xd, gd, sd = x.to(DEV), g.to(DEV), scale.to(DEV)
    dw, db = engine.conv_wgrad_ex(gd, xd, cout, ksize, stride, None, 0, bias=False, row_scale=sd)
    assert db is None
    dw2, _ = engine.conv_wgrad_ex(gd, xd, cout, ksize, stride, None, 0, bias=False, row_scale=sd)
    assert torch.equal(dw, dw2)
    plain, _ = engine.conv_wgrad_ex(gd, xd, cout, ksize, stride, None, 0, bias=False)
    assert torch.equal(dw, plain * sd.view(-1, 1, 1, 1))                       # one fp32 multiply per element
    x64, g64 = x.double().permute(0, 3, 1, 2), g.double().permute(0, 3, 1, 2)
    ref = torch.nn.grad.conv2d_weight(x64, (cout, cin, ksize, ksize), g64, stride=stride, padding=ksize // 2)
    bound = torch.nn.grad.conv2d_weight(x64.abs(), (cout, cin, ksize, ksize), g64.abs(), stride=stride, padding=ksize // 2)
    err = ((plain.cpu().double() - ref).abs() / (bound * 2.0 ** -23 * 64 + 1e-30)).max()
    print("dense wgrad %s: worst %.3g of 64 * 2^-23 * sum|g x|" % ((n, h, w, cin, cout, ksize, stride), float(err)))
    assert float(err) < 1.0


@pytest.mark.parametrize("n,h,w,cin,cout,residual", [(2, 16, 24, 2048, 512, False), (2, 13, 21, 512, 1024, True),
                                                     (1, 25, 40, 256, 128, True), (3, 7, 9, 1024, 256, False)])
def test_masked_1x1_dgrad_vs_float64(n, h, w, cin, cout, residual):
    """The 1x1 input gradient: mask(x > 0) * (g W^T + residual) against float64 on the same fp16 operands."""
    from retinanet_examples_b200 import engine
    gen = torch.Generator().manual_seed(n + h + cin + cout)
    g = _rnd(gen, n, h, w, cin, scale=0.1)
    wt = torch.randn((cin, cout, 1, 1), generator=gen) * 0.05
    mask = _rnd(gen, n, h, w, cout)
    res = _rnd(gen, n, h, w, cout) if residual else None
    out = engine.conv2d_dgrad(g.to(DEV), engine.pack_weight_dgrad(wt.to(DEV), cin), cout, mask=mask.to(DEV),
                              residual=res.to(DEV) if residual else None).cpu()
    ref = g.double().reshape(-1, cin) @ wt.half().double().reshape(cin, cout)
    if residual:
        ref = ref + res.double().reshape(-1, cout)
    ref = torch.where(mask.reshape(-1, cout) > 0, ref, torch.zeros_like(ref)).reshape(out.shape)
    assert bool((out[mask <= 0] == 0).all())
    err = float((out.double() - ref).abs().max() / ref.abs().max())
    print("1x1 dgrad %s: worst %.3g of max|ref|" % ((n, h, w, cin, cout, residual), err))
    assert err < 2e-3


def test_dilate_into_is_bit_exact():
    """An atlas level copied into a dense tensor (stride 1) and a dense gradient scattered to the even positions of a
    stride-2 layer's input (stride 2): bit-exact, nothing else written."""
    from retinanet_examples_b200 import engine
    gen = torch.Generator().manual_seed(3)
    src = _rnd(gen, 2, 40, 24, 256).to(DEV)
    dst = torch.full((2, 7, 11, 256), 7.0, dtype=torch.float16, device=DEV)
    engine.dilate_into(src, (17, 7, 11), dst, 1)
    assert torch.equal(dst, src[:, 17:24, :11])
    g = _rnd(gen, 2, 7, 11, 512).to(DEV)
    z = torch.zeros((2, 13, 21, 512), dtype=torch.float16, device=DEV)
    engine.dilate_into(g, (0, 7, 11), z, 2)
    ref = torch.zeros_like(z)
    ref[:, 0::2, 0::2] = g
    assert torch.equal(z, ref)


def _ref_stage_grads(m, params, st, fp16):
    """CPU fp32 autograd of the oracle's layer3 / layer4 blocks (from the model's own saved C3 -- or C4 in scope
    "layer4"), FPN and heads, times the model's own loss gradients; returns the gradients of `params`."""
    from oracle import model_ref
    from oracle.model_ref import _cb, _q
    import torch.nn.functional as F
    S = st["fpn"]
    blocks = m._backbone_blocks()
    sd = dict(m._sd)
    ref = {k: p.detach().cpu().clone().requires_grad_(True) for k, p in params.items()}
    sd.update(ref)
    bottleneck = len(blocks[0][1]["convs"]) == 3
    taps = {}
    x = S["c3" if blocks[0][1]["level"] == 4 else "c4"].permute(0, 3, 1, 2).float().cpu()
    for _, blk in blocks:
        p = blk["name"] + "."
        stride = blk["convs"][1 if bottleneck else 0]["stride"]
        if bottleneck:
            out = _q(F.relu(_cb(sd, p + "conv1", p + "bn1", x, 1, 0, fp16)), fp16)
            out = _q(F.relu(_cb(sd, p + "conv2", p + "bn2", out, stride, 1, fp16)), fp16)
            out = _cb(sd, p + "conv3", p + "bn3", out, 1, 0, fp16)
        else:
            out = _q(F.relu(_cb(sd, p + "conv1", p + "bn1", x, stride, 1, fp16)), fp16)
            out = _cb(sd, p + "conv2", p + "bn2", out, 1, 1, fp16)
        identity = _q(_cb(sd, p + "downsample.0", p + "downsample.1", x, stride, 0, fp16), fp16) if blk["down"] else x
        x = _q(F.relu(out + identity), fp16)
        taps[blk["level"]] = x
    c3 = S["c3"].permute(0, 3, 1, 2).float().cpu()
    c4 = taps.get(4, S["c4"].permute(0, 3, 1, 2).float().cpu())
    feats = model_ref._fpn(sd, m.backbone, c3, c4, taps[5], fp16)
    total = 0.0
    for head in ("cls_head", "box_head"):
        for l, f in enumerate(feats):
            total = total + (model_ref.head(sd, head, f, fp16=fp16) * st["grads"][head][l].cpu()).sum()
    total.backward()
    return {k: v.grad for k, v in ref.items()}


@pytest.mark.parametrize("backbone,rotated,shape", [("ResNet18FPN", False, (2, 256, 384)), ("ResNet18FPN", True, (2, 256, 384)),
                                                    ("ResNet50FPN", False, (2, 256, 384)), ("ResNet50FPN", True, (2, 256, 384)),
                                                    ("ResNet50FPN", False, (1, 800, 1280))])
def test_model_stage_gradients_vs_cpu_autograd(backbone, rotated, shape):
    """Every layer3 / layer4 weight gradient of scope "layer3" against CPU fp32 autograd and the fp16-emulating oracle
    run from the model's own saved C3 and loss gradients, per tensor relative to max|ref|, bar 5e-2 (loss scaled by
    2^16).  The measured worst values are printed and recorded in DESIGN.md."""
    from retinanet_examples_b200.model import Model, make_state_dict
    m = Model(backbone, classes=3, rotated_bbox=rotated)
    m.load_state_dict(_lively(make_state_dict(backbone, 3, m.num_anchors, rotated, seed=4), 11)).cuda(0)
    m.set_train_scope("layer3")
    params = dict(m.named_parameters())
    bb = m._backbone_param_names()
    m.train()
    m.want_atlas_grad = True
    g = torch.Generator().manual_seed(12)
    n, H, W = shape
    x = torch.randn((n, 3, H, W), generator=g).to(DEV)
    t = _targets(n, rotated, g, (H, W)).to(DEV)
    cls_loss, box_loss = m([x, t])
    ((cls_loss + box_loss) * 2.0 ** 16).backward()
    st = m.last_train
    sub = {k: params[k] for k in bb}
    for tag, fp16 in (("fp32", False), ("fp16-emulating", True)):
        ref = _ref_stage_grads(m, sub, st, fp16)
        e = {k: float((sub[k].grad.cpu() / 2.0 ** 16 - ref[k]).abs().max() / ref[k].abs().max()) for k in bb}
        worst = max(e, key=e.get)
        print("model %s %s %s vs the %s oracle: worst %s %.3g" % (backbone, "rotated" if rotated else "axis", shape, tag,
                                                                  worst, e[worst]))
        for k, v in e.items():
            assert v < 5e-2, (tag, k, v)


def test_stage_gradients_match_the_reference_golden(golden_dir):
    """The unmodified reference's training-mode ResNet18FPN on the CPU in fp32 (oracle/gen_golden_backbone_grads.py)
    against this model in scope "layer3": the losses, the stored output channels and the per-channel gradient norms of
    every layer3 / layer4 weight within 5e-2 * max|ref| per tensor, and the reference's parameter order."""
    from oracle.gen_golden_backbone_grads import BACKBONE, CLASSES, inputs, stage_weight
    from retinanet_examples_b200.model import Model
    gd = np.load(os.path.join(golden_dir, "backbone_grads.npz"))
    sd, x, t = inputs()
    m = Model(BACKBONE, classes=CLASSES).load_state_dict(sd).cuda(0).set_train_scope("layer3")
    params = dict(m.named_parameters())
    names = [str(n) for n in gd["names"]]
    assert list(params) == [n for n in names if stage_weight(n) and n.endswith("weight") and ".bn" not in n
                            and ".downsample.1." not in n] + [n for n in names if ".features." not in n and n.startswith("backbones")] + \
        [n for n in names if not n.startswith("backbones")]
    m.train()
    cls_loss, box_loss = m([x.to(DEV), t.to(DEV)])
    ((cls_loss + box_loss) * 2.0 ** 16).backward()
    errs = {"cls_loss": abs(float(cls_loss) / float(gd["cls_loss"]) - 1), "box_loss": abs(float(box_loss) / float(gd["box_loss"]) - 1)}
    for name in m._backbone_param_names():
        gw = params[name].grad.cpu() / 2.0 ** 16
        ch = torch.from_numpy(gd[name + ".channels"]).long()
        for tag, a, r in (("w", gw[ch], gd[name]), ("norm", gw.flatten(1).norm(dim=1), gd[name + ".norms"])):
            r = torch.from_numpy(r)
            errs[name + "." + tag] = float((a - r).abs().max() / r.abs().max())
    worst = max(errs, key=errs.get)
    print("golden backbone grads: worst %s %.3g; losses %.3g / %.3g" % (worst, errs[worst], errs["cls_loss"], errs["box_loss"]))
    for k, v in errs.items():
        assert v < 5e-2, (k, v)


def _model(scope, seed=6):
    from retinanet_examples_b200.model import Model, make_state_dict
    sd = _lively(make_state_dict("ResNet18FPN", 3, 9, False, seed=seed), seed)
    m = Model("ResNet18FPN", classes=3).load_state_dict(sd).cuda(0).set_train_scope(scope)
    g = torch.Generator().manual_seed(seed)
    return m, torch.randn((2, 3, 256, 384), generator=g).to(DEV), _targets(2, False, g, (256, 384)).to(DEV)


def _grads(m, x, t):
    m.zero_grad()
    m.train()
    cls_loss, box_loss = m([x, t])
    ((cls_loss + box_loss) * 1024.0).backward()
    return {k: (p.grad.clone() if p.grad is not None else None) for k, p in m.named_parameters()}


def test_parameters_order_identity_and_scope_equivalence():
    """named_parameters() follows _param_names() and keeps each tensor across scope changes; head and FPN gradients of
    scope "layer3" equal scope "fpn"'s bit for bit; with layer3 frozen, scope "layer3" equals scope "layer4"; two
    backwards are bit-identical."""
    m3, x, t = _model("layer3")
    p3 = dict(m3.named_parameters())
    assert list(p3) == m3._param_names()
    g3 = _grads(m3, x, t)
    assert all(g is not None and int(g.count_nonzero()) > 0 for g in g3.values())
    again = _grads(m3, x, t)
    for k in g3:
        assert torch.equal(g3[k], again[k]), k
    p_fpn = dict(m3.set_train_scope("fpn").named_parameters())
    assert all(p_fpn[k] is p3[k] for k in p_fpn)
    assert all(p is p3[k] for k, p in m3.set_train_scope("layer3").named_parameters())
    mf, _, _ = _model("fpn")
    gf = _grads(mf, x, t)
    for k in gf:
        assert torch.equal(gf[k], g3[k]), k
    m4, _, _ = _model("layer4")
    g4 = _grads(m4, x, t)
    for k in m3._param_names():
        if ".layer3." in k:
            p3[k].requires_grad_(False)
    g3f = _grads(m3, x, t)
    for k, v in g4.items():
        assert torch.equal(g3f[k], v), k


def test_training_loop_sgd_gradscaler_layer3_scope():
    """20 iterations of the reference's loop (SGD with momentum and weight decay, LambdaLR warm-up, GradScaler) in scope
    "layer3" on ResNet18FPN: every step's loss within 1e-2 (relative) of a CPU fp32 run of the same steps (the oracle's
    layer3-4, FPN and heads on the model's frozen C3), the stem, layer1, layer2 and every BN buffer bit-identical while the
    layer3 / layer4 weights change, fp16 / fp32 / INT8-network eval equal a fresh model loaded from state_dict(), and a
    2^40 loss scale skips the step."""
    from oracle import model_ref
    from retinanet_examples_b200.model import Model, make_state_dict
    import torch.nn.functional as F
    from oracle.model_ref import _cb
    classes = 3
    sd = make_state_dict("ResNet18FPN", classes, 9, False, seed=6)
    m = Model("ResNet18FPN", classes=classes).load_state_dict(sd).cuda(0).set_train_scope("layer3")
    names = m._param_names()
    frozen = {k: v.clone() for k, v in sd.items() if k not in set(names)}
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
    blocks = m._backbone_blocks()

    def ref_forward(c3):
        x, taps = c3, {}
        for _, blk in blocks:
            p, s = blk["name"] + ".", blk["convs"][0]["stride"]
            out = _cb(ref_sd, p + "conv2", p + "bn2", F.relu(_cb(ref_sd, p + "conv1", p + "bn1", x, s, 1)), 1, 1)
            ident = _cb(ref_sd, p + "downsample.0", p + "downsample.1", x, s, 0) if blk["down"] else x
            x = taps[blk["level"]] = F.relu(out + ident)
        return model_ref._fpn(ref_sd, "ResNet18FPN", c3, taps[4], taps[5], False)

    m.want_atlas_grad = True
    m.train()
    losses, ref_losses, cache = [], [], {}
    for it in range(20):
        x, t = data[it % 2]
        opt.zero_grad()
        cls_loss, box_loss = m([x, t])
        if it % 2 not in cache:
            views = m.last_train["views"]
            tg = [m._extract_targets(t, x.shape[-1] // v.w, (v.h, v.w)) for v in views]
            cache[it % 2] = (m.last_train["fpn"]["c3"].permute(0, 3, 1, 2).float().cpu(), [a.cpu() for a, _, _ in tg],
                             [b.cpu() for _, b, _ in tg])
        scaler.scale(cls_loss + box_loss).backward()
        before = scaler.get_scale()
        scaler.step(opt)
        scaler.update()
        skipped = scaler.get_scale() < before
        scheduler.step()
        losses.append(float((cls_loss + box_loss).detach()))
        c3, ci, bt = cache[it % 2]
        ref_opt.zero_grad()
        feats = ref_forward(c3)
        rc, rb = _cpu_loss([model_ref.head(ref_sd, "cls_head", f) for f in feats],
                           [model_ref.head(ref_sd, "box_head", f) for f in feats], ci, bt, classes)
        (rc + rb).backward()
        if not skipped:
            ref_opt.step()
        ref_sched.step()
        ref_losses.append(float((rc + rb).detach()))
    dev = max(abs(a - b) / b for a, b in zip(losses, ref_losses))
    print("layer3 scope losses", [round(v, 4) for v in losses])
    print("cpu fp32 losses", [round(v, 4) for v in ref_losses], "worst relative difference %.3g" % dev)
    assert all(math.isfinite(v) for v in losses)
    assert dev < 1e-2, dev
    m.want_atlas_grad = False
    trained = m.state_dict()
    for k, v in frozen.items():
        assert torch.equal(trained[k], v), k
    for k in m._backbone_param_names():
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
