"""One small launch of every kernel variant of the hot path, for compute-sanitizer:
    compute-sanitizer --tool memcheck  python tools/sanitize_cases.py
    compute-sanitizer --tool racecheck python tools/sanitize_cases.py
    compute-sanitizer --tool synccheck python tools/sanitize_cases.py
Shapes are tiny (the tools slow kernels down 10-100x) but chosen to reach each variant of the wgmma kernels and their
mbarrier rings: conv modes 0 / 1 / 2 / 3 with N tiles 64 and 128, ragged M and N tiles, residual / upsample / ReLU6 /
fp32 / sigmoid / candidate epilogues, the fused stem + pool (stem.cu: halo rows at the image edges), the fused bottleneck
tail (bottleneck.cu: C1 64 / 128, projected identity, GEMM3 with 64 / 128 outputs -- shared-memory A operands written
by the epilogues), decode (filter / gather / select), NMS (shared-memory aliasing of the sort scratch), rotated NMS,
iou, target assignment, the cooperative loss kernel."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from retinanet_examples_b200 import _C, box, engine, loss, synth  # noqa: E402
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


def main():
    only = sys.argv[1] if len(sys.argv) > 1 else ""
    if only in ("", "conv"):
        conv(2, 16, 16, 64, 64, 1, relu=True)                              # mode 0
        conv(2, 16, 16, 256, 256, 1, relu=True, residual=True)             # residual epilogue
        conv(1, 16, 32, 256, 256, 1, upsample=True)                        # upsample-add epilogue
        conv(1, 18, 20, 256, 256, 1, upsample=True)                        # ragged last M tile
        conv(1, 16, 24, 64, 64, 3, relu=True)                              # mode 1, N tile 64
        conv(1, 7, 10, 256, 256, 3, relu=True)                             # mode 1, patch of 70 pixels
        conv(10, 48, 64, 256, 256, 3, relu=True)                           # mode 1, N tile 128, several tiles per CTA
        conv(2, 100, 160, 256, 36, 3, out_mode=engine.OUT_NCHW_F32)        # narrow head output, ragged N tile
        conv(1, 24, 32, 256, 720, 3, out_mode=engine.OUT_NCHW_F32_SIGMOID)
        conv(2, 26, 40, 128, 128, 3, relu=True, stride=2)                  # parity-split stride 2
        conv(2, 25, 39, 256, 256, 3, relu=True, stride=2)                  # element-strided boxes
        conv(40, 100, 160, 64, 256, 1, relu=True)                          # enough tiles for 1x1
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
    if only in ("", "model"):
        for rotated in (False, True):
            classes, na = 4, 27 if rotated else 9
            sd = make_state_dict("ResNet18FPN", classes, na, rotated, seed=1)
            sd["cls_head.8.bias"] = torch.full_like(sd["cls_head.8.bias"], -2.5)
            m = Model("ResNet18FPN", classes=classes, rotated_bbox=rotated).load_state_dict(sd).cuda(0)
            out = m(torch.randn((2, 3, 128, 256), generator=g).to(DEV))     # fused candidate epilogue -> decode -> nms
            torch.cuda.synchronize()
            print("model rotated=%s detections=%d" % (rotated, int((out[0] > 0).sum())), flush=True)
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


if __name__ == "__main__":
    main()
