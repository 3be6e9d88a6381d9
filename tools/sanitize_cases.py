"""One small launch of every kernel variant of the hot path, for compute-sanitizer:
    compute-sanitizer --tool memcheck  python tools/sanitize_cases.py
    compute-sanitizer --tool racecheck python tools/sanitize_cases.py
    compute-sanitizer --tool synccheck python tools/sanitize_cases.py
Shapes are tiny (the tools slow kernels down 10-100x) but chosen to reach each variant of the wgmma kernels and their
mbarrier rings: conv modes 0 / 1 / 2 / 3 with N tiles 64 and 128 (and 256 in modes 0 / 1), ragged M and N tiles, residual / upsample / ReLU6 /
fp32 / sigmoid / candidate epilogues, the fused stem + pool (stem.cu: halo rows at the image edges), the fused bottleneck
tail (bottleneck.cu: C1 64 / 128, projected identity, GEMM3 with 64 / 128 outputs -- shared-memory A operands written
by the epilogues), the s8 instantiation of the conv kernel (stride 2 in modes 3 and 1, residual / upsample addends, level-view
input and output) and the INT8 heads and network scope of the model, the split-TF32 fp32 instantiation (`fp32`: modes 0 / 1 / 2 /
3, N tiles 64 / 128, several tiles per CTA so the A_lo side buffers and the named barrier cycle, tile table and level views,
fp32 addends, NCHW / sigmoid / candidate epilogues, the fp32 small kernels, the fp32 model), decode (filter / gather / select), NMS (shared-memory aliasing of the sort scratch), rotated NMS,
iou, target assignment, the cooperative loss kernel, and head training (`train`: the weight-gradient kernel, the bias-gradient
and reduce kernels, the gradient atlas, the masked input-gradient conv instance, one SGD step of the model), and FPN
training (`train_fpn`: the wgrad_ex instance in its three modes, the level bias-gradient and 1-tap reduce kernels, the
pool-add and dilation kernels, one SGD step of the model in the "fpn" scope)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from retinanet_examples_b200 import _C, _lib, box, engine, loss, synth  # noqa: E402
from retinanet_examples_b200.model import Model, make_state_dict  # noqa: E402

DEV = "cuda:0"
g = torch.Generator().manual_seed(0)


def rnd(*shape, scale=1.0):
    return (torch.randn(shape, generator=g) * scale).to(torch.float16).to(DEV)


def conv(n, h, w, cin, cout, ks, **kw):
    x, wt, b = rnd(n, h, w, cin), engine.pack_weight(torch.randn((cout, cin, ks, ks), generator=g) * 0.05).to(DEV), torch.randn(cout, generator=g).to(DEV)
    res = rnd(n, h, w, cout) if kw.pop("residual", False) else None
    up = rnd(n, h // 2, w // 2, cout) if kw.pop("upsample", False) else None
    y = engine.conv2d(x, wt, b, cout, ks, residual=res, upsample=up, **kw)
    torch.cuda.synchronize()
    print("conv %s -> plan %s" % ((n, h, w, cin, cout, ks), {k: v for k, v in engine.last_plan().items() if v}), flush=True)
    return y


def conv32(n, h, w, cin, cout, ks, x=None, **kw):
    """One odtk_conv2d_f32 launch on random fp32 operands (addends requested by residual=True / upsample=True)."""
    x = (torch.randn((n, h, w, cin), generator=g).to(DEV)) if x is None else x
    hi, lo = [t.to(DEV) for t in engine.pack_weight_tf32x2(torch.randn((cout, cin, ks, ks), generator=g) * 0.05)]
    stride = kw.get("stride", 1)
    oh, ow = ((h - 1) // 2 + 1, (w - 1) // 2 + 1) if stride == 2 else (h, w)
    if kw.pop("residual", False):
        kw["residual"] = torch.randn((n, oh, ow, cout), generator=g).to(DEV)
    if kw.pop("upsample", False):
        kw["upsample"] = torch.randn((n, h // 2, w // 2, cout), generator=g).to(DEV)
    y = engine.conv2d_f32(x, hi, lo, torch.randn(cout, generator=g).to(DEV), cout, ks, **kw)
    torch.cuda.synchronize()
    print("conv_f32 %s -> plan %s" % ((n, h, w, cin, cout, ks, stride), {k: v for k, v in engine.last_plan().items() if v}), flush=True)
    return y


def fp32_cases():
    """Every variant of the split-TF32 instance (conv.cu, kOpTF32x3) and the fp32 twins of layers.cu."""
    conv32(2, 16, 16, 64, 64, 1, relu=True)                                # mode 0, N tile 64
    conv32(2, 16, 16, 256, 256, 1, relu=True, residual=True)               # residual epilogue
    conv32(1, 16, 32, 256, 256, 1, upsample=True)                          # upsample-add epilogue
    conv32(1, 18, 20, 256, 256, 1, upsample=True)                          # ragged last M tile
    conv32(40, 100, 160, 64, 256, 1, relu=True)                            # mode 0, N tile 128, several tiles per CTA
    conv32(1, 16, 24, 64, 64, 3, relu=True)                                # mode 1, N tile 64
    conv32(1, 7, 10, 96, 256, 3, relu=True)                                # mode 1, 70-pixel patch, 3 K blocks per tap
    conv32(10, 48, 64, 256, 256, 3, relu=True, residual=True)              # mode 1, N tile 128, several tiles per CTA
    conv32(2, 26, 40, 128, 128, 3, relu=True, stride=2)                    # mode 3 (parity split)
    conv32(2, 28, 20, 256, 512, 1, stride=2)                               # mode 3, 1x1
    conv32(2, 25, 39, 256, 256, 3, relu=True, stride=2)                    # mode 1, element-strided boxes
    conv32(2, 100, 160, 256, 36, 3, out_mode=engine.OUT_NCHW_F32)          # narrow head output, ragged N tile
    conv32(1, 24, 32, 256, 720, 3, out_mode=engine.OUT_NCHW_F32_SIGMOID)   # ragged 128-wide N tile
    conv32(1, 5, 7, 256, 2160, 3, out_mode=engine.OUT_NCHW_F32)
    # stem (mode 2) over the fp32 NHWC4 image: even and odd sides; max-pool
    for h, w in ((64, 96), (37, 51)):
        x = torch.randn((2, h, w, 3), generator=g).to(DEV)
        hi, lo = [t.to(DEV) for t in engine.pack_stem_weight_tf32x2(torch.randn((64, 3, 7, 7), generator=g) * 0.1)]
        engine.maxpool3x3s2_f32(engine.stem_conv_f32(engine.pad_input_f32(x), h, w, hi, lo, torch.randn(64, generator=g).to(DEV), 64))
        torch.cuda.synchronize()
        print("stem_f32 %dx%d ok" % (h, w), flush=True)
    # atlas: one launch over every level (tile table), level view -> level view, stride 2 into a level view, ReLU copy
    m = Model("ResNet18FPN", classes=2)
    sizes = ((20, 32), (10, 16), (5, 8), (3, 4), (2, 2))
    at = m._atlas_for(2, sizes, torch.device(DEV))
    xa = torch.randn(at["buf"][0].shape, generator=g).to(DEV)
    ya = torch.zeros(at["buf"][0].shape, dtype=torch.float32, device=DEV)
    conv32(2, xa.shape[1], xa.shape[2], 256, 256, 3, x=xa, relu=True, out=ya, tile_tab=at["tab"])
    conv32(2, *sizes[1], 256, 256, 3, x=engine.AtlasView(xa, at["rows"][1], *sizes[1]), out=engine.AtlasView(ya, at["rows"][1], *sizes[1]))
    conv32(2, *sizes[2], 256, 256, 3, stride=2, out=engine.AtlasView(ya, at["rows"][3], *sizes[3]))
    engine.relu_from_view(engine.AtlasView(ya, at["rows"][3], *sizes[3]))
    # input side
    engine.preprocess_u8_f32(torch.randint(0, 256, (2, 100, 130, 3), dtype=torch.uint8, generator=g).to(DEV))
    imgs = [torch.randint(0, 256, s, dtype=torch.uint8, generator=g) for s in ((30, 40, 3), (300, 170, 3), (900, 41, 3))]
    engine.preprocess_resize_u8(imgs, 64, 100, f32=True)
    torch.cuda.synchronize()
    print("fp32 layers ok", flush=True)
    # the fp32 model: candidate epilogue and dense route, axis-aligned and rotated
    for rotated in (False, True):
        classes, na = 4, 27 if rotated else 9
        sd = make_state_dict("ResNet18FPN", classes, na, rotated, seed=1)
        sd["cls_head.8.bias"] = torch.full_like(sd["cls_head.8.bias"], -2.5)
        m = Model("ResNet18FPN", classes=classes, rotated_bbox=rotated).load_state_dict(sd).cuda(0).set_precision("fp32")
        x = torch.randn((2, 3, 128, 256), generator=g).to(DEV)
        for fused in (True, False):
            m.fused_candidates = fused
            out = m(x)
            torch.cuda.synchronize()
            print("model fp32 rotated=%s fused=%s detections=%d" % (rotated, fused, int((out[0] > 0).sum())), flush=True)


def train_cases():
    """Head training: wgrad_kernel (TMA / mbarrier ring, split-K partial writes, an output tile with no second 64-channel
    G box, a dense image without tile table), bgrad_partial / wgrad_reduce, grad_to_atlas_kernel, the kOpF16Mask conv
    instance with its mask and residual reads in tile-table mode, and one SGD step of the model."""
    from retinanet_examples_b200.model import Model as M
    at = M("ResNet18FPN", classes=1)._atlas_for(2, ((16, 24), (8, 12), (4, 6), (2, 3), (1, 2)), torch.device(DEV))
    n, ha, wa = at["buf"][0].shape[:3]
    for cout in (256, 36):
        cpad = engine.pad64(cout)
        gg, xx = rnd(n, ha, wa, cpad, scale=0.1), rnd(n, ha, wa, 256)
        engine.conv_wgrad(gg, xx, cout, tile_tab=at["tab"])
        engine.conv_wgrad(gg, xx, cout)
        wd = engine.pack_weight_dgrad(torch.randn((cout, 256, 3, 3), generator=g).to(DEV) * 0.02, cpad)
        a = engine.conv2d_dgrad(gg, wd, 256, mask=xx, tile_tab=at["tab"])
        engine.conv2d_dgrad(gg, wd, 256, residual=a, tile_tab=at["tab"])
        torch.cuda.synchronize()
        print("wgrad / dgrad cout=%d ok" % cout, flush=True)
    grads = [torch.randn((2, 54, h, w), generator=g).to(DEV) for h, w in ((16, 24), (8, 12), (4, 6), (2, 3), (1, 2))]
    engine.grad_to_atlas(grads, at["rows"], 3.0, torch.zeros((n, ha, wa, 64), dtype=torch.float16, device=DEV))
    sd = make_state_dict("ResNet18FPN", 3, 9, False, seed=1)
    m = Model("ResNet18FPN", classes=3).load_state_dict(sd).cuda(0)
    opt = torch.optim.SGD(m.parameters(), lr=0.01, momentum=0.9)
    m.train()
    x = torch.randn((2, 3, 128, 256), generator=g).to(DEV)
    t = torch.tensor([[[20., 30., 60., 40., 1.], [100., 10., 50., 90., 2.]], [[5., 5., 100., 100., 0.], [-1.] * 5]]).to(DEV)
    cls_loss, box_loss = m([x, t])
    ((cls_loss + box_loss) * 1024.0).backward()
    opt.step()
    torch.cuda.synchronize()
    print("train step ok", flush=True)


def train_fpn_cases():
    """FPN training: wgrad_kernel through odtk_conv_wgrad_ex (1x1, 3x3 stride 1, 3x3 stride 2 element-strided boxes, a
    level at a nonzero g_row0, odd level sizes), bgrad_level_partial / wgrad_reduce<1>, pool_add (pool 2 in place with a
    missing source row, pool 1), dilate, and one SGD step of the model in the "fpn" scope."""
    sizes = ((16, 24), (8, 12), (7, 10), (4, 5), (2, 3))
    at = Model("ResNet18FPN", classes=1)._atlas_for(2, sizes, torch.device(DEV))
    n, ha, wa = at["buf"][0].shape[:3]
    tabs = at["tabs"]
    gg = rnd(n, ha, wa, 256, scale=0.1)
    engine.conv_wgrad_ex(gg, rnd(n, 8, 12, 512), 256, 1, 1, tabs[1], at["rows"][1])
    engine.conv_wgrad_ex(gg, rnd(n, 7, 10, 256), 256, 3, 1, tabs[2], at["rows"][2])
    engine.conv_wgrad_ex(gg, rnd(n, 7, 10, 256), 256, 3, 2, tabs[3], at["rows"][3], bias=False)
    engine.conv_wgrad_ex(gg, rnd(n, 4, 5, 128), 256, 3, 2, tabs[4], at["rows"][4])
    torch.cuda.synchronize()
    print("wgrad_ex ok", flush=True)
    lv = [(r, h, w) for r, (h, w) in zip(at["rows"], sizes)]
    engine.pool_add(gg, gg, lv[0], lv[1], pool=2)
    engine.pool_add(gg, gg, lv[3], lv[4], pool=2)
    engine.pool_add(rnd(n, ha, wa, 256), gg, lv[2], lv[2], pool=1)
    engine.dilate(gg, torch.zeros_like(gg), lv[4], at["rows"][3])
    torch.cuda.synchronize()
    print("pool_add / dilate ok", flush=True)
    m = Model("ResNet18FPN", classes=3).load_state_dict(make_state_dict("ResNet18FPN", 3, 9, False, seed=1)).cuda(0)
    opt = torch.optim.SGD(m.set_train_scope("fpn").parameters(), lr=0.01, momentum=0.9)
    m.train()
    x = torch.randn((2, 3, 128, 256), generator=g).to(DEV)
    t = torch.tensor([[[20., 30., 60., 40., 1.], [100., 10., 50., 90., 2.]], [[5., 5., 100., 100., 0.], [-1.] * 5]]).to(DEV)
    cls_loss, box_loss = m([x, t])
    ((cls_loss + box_loss) * 1024.0).backward()
    opt.step()
    torch.cuda.synchronize()
    print("train fpn step ok", flush=True)


def main():
    only = sys.argv[1] if len(sys.argv) > 1 else ""
    if only in ("", "train"):
        train_cases()
    if only in ("", "train_fpn"):
        train_fpn_cases()
    if only in ("", "conv"):
        conv(2, 16, 16, 64, 64, 1, relu=True)                              # mode 0
        conv(2, 16, 16, 256, 256, 1, relu=True, residual=True)             # residual epilogue
        conv(1, 16, 32, 256, 256, 1, upsample=True)                        # upsample-add epilogue
        conv(1, 18, 20, 256, 256, 1, upsample=True)                        # ragged last M tile
        conv(1, 16, 24, 64, 64, 3, relu=True)                              # mode 1, N tile 64
        conv(1, 7, 10, 256, 256, 3, relu=True)                             # mode 1, patch of 70 pixels
        conv(10, 48, 64, 256, 256, 3, relu=True)                           # mode 1, N tile 128, several tiles per CTA
        _lib.lib().odtk_set_sm_budget(2)                                   # N tile 256: a 2-SM budget makes few tiles enough
        try:
            conv(2, 48, 64, 256, 256, 3, relu=True)                        # mode 1, several tiles per CTA
            conv(1, 32, 48, 256, 720, 3, out_mode=engine.OUT_NCHW_F32_SIGMOID)   # ragged third N tile
            conv(1, 50, 60, 512, 1024, 1, relu=True, residual=True)        # mode 0, ragged last M tile, residual
        finally:
            _lib.lib().odtk_set_sm_budget(0)
        conv(2, 100, 160, 256, 36, 3, out_mode=engine.OUT_NCHW_F32)        # narrow head output, ragged N tile
        conv(1, 24, 32, 256, 720, 3, out_mode=engine.OUT_NCHW_F32_SIGMOID)
        conv(2, 26, 40, 128, 128, 3, relu=True, stride=2)                  # parity-split stride 2
        conv(2, 25, 39, 256, 256, 3, relu=True, stride=2)                  # element-strided boxes
        conv(40, 100, 160, 64, 256, 1, relu=True)                          # enough tiles for 1x1
        _lib.lib().odtk_set_tma_store(0)                                   # the direct-store epilogues
        try:
            conv(2, 16, 16, 256, 256, 1, relu=True, residual=True)
            conv(1, 7, 10, 256, 256, 3, relu=True)
        finally:
            _lib.lib().odtk_set_tma_store(1)
        for c1, proj in ((64, False), (128, False), (64, True)):           # fused bottleneck tail: residual / streamed weights / projected identity
            c2 = 4 * c1
            xx, w2 = rnd(3, 9, 17, c1), engine.pack_weight(torch.randn((c1, c1, 3, 3), generator=g) * 0.05).to(DEV)
            w3 = engine.pack_weight(torch.randn((c2, c1, 1, 1), generator=g) * 0.05).to(DEV)
            b2, b3 = torch.randn(c1, generator=g).to(DEV), torch.randn(c2, generator=g).to(DEV)
            if proj:
                engine.bottleneck_tail(xx, w2, b2, w3, b3, None, xproj=rnd(3, 9, 17, 64), wproj=engine.pack_weight(torch.randn((c2, 64, 1, 1), generator=g) * 0.05).to(DEV))
            else:
                engine.bottleneck_tail(xx, w2, b2, w3, b3, rnd(3, 9, 17, c2))
            torch.cuda.synchronize()
            print("bottleneck_tail c1=%d proj=%s ok" % (c1, proj), flush=True)
        for c3 in (64, 128):                                               # + GEMM3: the next block's conv1 from the block output
            xx, w2 = rnd(3, 9, 17, 64), engine.pack_weight(torch.randn((64, 64, 3, 3), generator=g) * 0.05).to(DEV)
            w3 = engine.pack_weight(torch.randn((256, 64, 1, 1), generator=g) * 0.05).to(DEV)
            wn = engine.pack_weight(torch.randn((c3, 256, 1, 1), generator=g) * 0.05).to(DEV)
            engine.bottleneck_tail(xx, w2, torch.randn(64, generator=g).to(DEV), w3, torch.randn(256, generator=g).to(DEV), rnd(3, 9, 17, 256),
                                   w_next=wn, b_next=torch.randn(c3, generator=g).to(DEV))
            torch.cuda.synchronize()
            print("bottleneck_tail + next conv1 (%d) ok" % c3, flush=True)
        engine.depthwise3x3(rnd(2, 9, 11, 192), rnd(9, 192), torch.randn(192, generator=g).to(DEV), stride=2, act=2)
        conv(1, 48, 48, 192, 960, 1, relu=2)                               # ReLU6, ragged last 128-wide N tile
        torch.cuda.synchronize()
        x = rnd(2, 64, 96, 3)
        wt, b = engine.pack_stem_weight(torch.randn((64, 3, 7, 7), generator=g) * 0.1).to(DEV), torch.randn(64, generator=g).to(DEV)
        engine.stem_pool(x, wt, b, 64)
        engine.maxpool3x3s2(engine.stem_conv(x, wt, b, 64))
        engine.relu(rnd(2, 13, 20, 256))
        torch.cuda.synchronize()
        print("stem ok", flush=True)
        # s8 kernel: N tiles 64 / 128, s8 NHWC requantising epilogue, fp32 sigmoid epilogue with a ragged N tile, 1x1 rows
        for n, h, w, cin, cout, ks, mode in ((1, 16, 24, 256, 256, 3, engine.OUT_NHWC_S8), (10, 48, 64, 256, 256, 3, engine.OUT_NHWC_S8),
                                             (1, 13, 20, 256, 720, 3, engine.OUT_NCHW_F32_SIGMOID), (2, 16, 24, 128, 64, 1, engine.OUT_NHWC_S8)):
            xq = engine.quantize_f16_s8(rnd(n, h, w, cin), 20.0)
            wq, s_w = engine.pack_weight_s8(torch.randn((cout, cin, ks, ks), generator=g) * 0.05)
            engine.conv2d_s8(xq, wq.to(DEV), (s_w * 0.05).to(DEV), torch.randn(cout, generator=g).to(DEV), cout, ks,
                             relu=mode == engine.OUT_NHWC_S8, out_mode=mode, inv_out_scale=0.1)
            torch.cuda.synchronize()
            print("conv_s8 %s -> plan %s" % ((n, h, w, cin, cout, ks), {k: v for k, v in engine.last_plan().items() if v}), flush=True)
        # s8 network-scope paths: stride 2 (parity split / element-strided boxes), residual and upsample addends, s8 atlas
        # level views in and out, ReLU copy of a level
        for n, h, w, cin, cout, ks, stride, add in ((2, 16, 24, 256, 256, 3, 2, ""), (2, 16, 24, 512, 256, 1, 2, ""),
                                                    (2, 13, 20, 256, 256, 3, 2, ""), (2, 16, 24, 256, 512, 1, 1, "res"),
                                                    (2, 16, 24, 256, 256, 3, 1, "res"), (2, 16, 24, 256, 256, 1, 1, "up")):
            xq = engine.quantize_f16_s8(rnd(n, h, w, cin), 20.0)
            oh, ow = ((h - 1) // 2 + 1, (w - 1) // 2 + 1) if stride == 2 else (h, w)
            wq, s_w = engine.pack_weight_s8(torch.randn((cout, cin, ks, ks), generator=g) * 0.05)
            kw = {"residual": engine.quantize_f16_s8(rnd(n, oh, ow, cout), 20.0), "res_scale": 0.05} if add == "res" else \
                 {"upsample": engine.quantize_f16_s8(rnd(n, oh // 2, ow // 2, cout), 20.0), "up_scale": 0.05} if add == "up" else {}
            engine.conv2d_s8(xq, wq.to(DEV), (s_w * 0.05).to(DEV), torch.randn(cout, generator=g).to(DEV), cout, ks, relu=True,
                             inv_out_scale=0.1, stride=stride, **kw)
            torch.cuda.synchronize()
            print("conv_s8_ex %s -> plan %s" % ((n, h, w, cin, cout, ks, stride, add), {k: v for k, v in engine.last_plan().items() if v}), flush=True)
        at = torch.zeros((2, 56, 24, 256), dtype=torch.int8, device=DEV)
        at[:, :32] = engine.quantize_f16_s8(rnd(2, 32, 24, 256), 20.0)
        wq, s_w = engine.pack_weight_s8(torch.randn((256, 256, 3, 3), generator=g) * 0.05)
        engine.conv2d_s8(engine.AtlasView(at, 0, 32, 24), wq.to(DEV), (s_w * 0.05).to(DEV), None, 256, 3, relu=True, stride=2,
                         out=engine.AtlasView(at, 40, 16, 12), inv_out_scale=0.1)
        engine.relu_from_view(engine.AtlasView(at, 40, 16, 12))
        torch.cuda.synchronize()
        print("conv_s8_ex atlas views ok", flush=True)
    if only in ("", "model"):
        for rotated in (False, True):
            classes, na = 4, 27 if rotated else 9
            sd = make_state_dict("ResNet18FPN", classes, na, rotated, seed=1)
            sd["cls_head.8.bias"] = torch.full_like(sd["cls_head.8.bias"], -2.5)
            m = Model("ResNet18FPN", classes=classes, rotated_bbox=rotated).load_state_dict(sd).cuda(0)
            x = torch.randn((2, 3, 128, 256), generator=g).to(DEV)
            out = m(x)                                                      # fused candidate epilogue -> decode -> nms
            torch.cuda.synchronize()
            print("model rotated=%s detections=%d" % (rotated, int((out[0] > 0).sum())), flush=True)
            m.set_precision("int8", m.calibrate([x], method="max"))       # INT8 heads: quantise, s8 towers over the atlas, s8 candidates
            out = m(x)
            torch.cuda.synchronize()
            print("model int8 rotated=%s detections=%d" % (rotated, int((out[0] > 0).sum())), flush=True)
            m.set_precision("int8", m.calibrate([x], method="max", scope="network"), scope="network")   # layer3/4 + FPN on s8
            out = m(x)
            torch.cuda.synchronize()
            print("model int8 network rotated=%s detections=%d" % (rotated, int((out[0] > 0).sum())), flush=True)
    if only in ("", "fp32"):
        fp32_cases()
    if only in ("", "postproc"):
        cls, deltas = synth.head_outputs(1, seed=0)
        anchors = [box.generate_anchors(s, box.DEFAULT_RATIOS, box.DEFAULT_SCALES).reshape(-1).tolist() for s in synth.LEVEL_STRIDES]
        dec = _C.decode_levels([c[:, :, :25, :40].contiguous().to(DEV) for c in cls[:3]], [d[:, :, :25, :40].contiguous().to(DEV) for d in deltas[:3]],
                               anchors[:3], synth.LEVEL_STRIDES[:3], 0.05, 1000)
        _C.nms(*dec, 0.5, 100)
        bq = torch.rand((5, 8), generator=g).to(DEV) * 50
        _C.iou(bq, torch.rand((300, 8), generator=g).to(DEV) * 50)
        torch.cuda.synchronize()
        print("postproc ok", flush=True)
    if only in ("", "loss"):
        t = torch.tensor([[[20., 30., 60., 40., 1.], [-1., -1., -1., -1., -1.]]]).to(DEV)
        anchors = box.generate_anchors(32, box.DEFAULT_RATIOS, box.DEFAULT_SCALES)
        _, bt, dp, ci = box.snap_to_anchors_batch(t, (8, 12), 32, anchors, 3, [0.4, 0.5], dense=False)
        c, b = torch.randn((1, 27, 8, 12), generator=g).to(DEV), torch.randn((1, 36, 8, 12), generator=g).to(DEV)
        loss.retina_loss([c], [b], [ci], [bt], 3, with_grad=True)
        torch.cuda.synchronize()
        print("loss ok", flush=True)
    if only in ("", "resize"):
        # raw-image resize into the stem buffer: an upscale, a downscale within the shared tap tables, one beyond them
        # (per-pixel taps), a same-size image and a tiny one, ragged in one canvas; CPU (staged) and CUDA (in place) input
        imgs = [torch.randint(0, 256, s, dtype=torch.uint8, generator=g) for s in ((30, 40, 3), (300, 170, 3), (900, 41, 3),
                                                                                    (64, 100, 3), (3, 5, 3))]
        engine.preprocess_resize_u8(imgs, 64, 100)
        engine.preprocess_resize_u8([i.to(DEV) for i in imgs], 64, 100, canvas=(256, 128))
        torch.cuda.synchronize()
        print("resize ok", flush=True)
    if only in ("", "jpeg"):
        # JPEG decode kernels (restart scan, entropy decode, IDCT, upsample + colour): every sampling, grayscale, restart
        # intervals, a 640x480 image, then a batch with a truncated stream (its decoder runs out of data and stops)
        import numpy as np
        fx = np.load(os.path.join(ROOT, "tests", "golden", "jpeg_pil.npz"))
        datas = [fx[n + "_jpeg"].tobytes() for n in ("420_q75", "422_restart_rows", "444_restart3", "gray_q100", "420_640x480",
                                                     "420_1x1")]
        engine.decode_jpeg(datas)
        _, status = engine.decode_jpeg(datas[:2] + [fx["truncated_jpeg"].tobytes()])
        torch.cuda.synchronize()
        print("jpeg ok status=%s" % status.cpu().tolist(), flush=True)


if __name__ == "__main__":
    main()
