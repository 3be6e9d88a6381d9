"""Head-training benchmark: ResNet50FPN at 800 x 1280, one SGD + GradScaler step of the head parameters (backbone and FPN
frozen).  Reports the step time split into forward (backbone, FPN, towers and final layers), loss (target assignment and the
fused loss launch) and backward (gradient atlas, weight and input gradients of the ten head layers), and per-launch
TFLOP/s of a tower layer's forward, weight-gradient and input-gradient launches over the pyramid atlas (CUDA events around
repeated launches, FLOPs = 2 * pixels of the levels * 256 * 9 * 256).
--scope fpn trains the FPN as well (Model.set_train_scope("fpn")) and reports the step split into forward, loss, head
backward (the same step with every FPN parameter frozen but d(atlas) computed) and FPN backward (the rest), and per
launch the time and TFLOP/s of each FPN layer's weight gradient (odtk_conv_wgrad_ex) next to its forward launch (FLOPs =
2 * output pixels * 256 * k^2 * Cin).
    python tools/train_heads_bench.py [--batch 8] [--steps 10] [--scope heads|fpn]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from retinanet_examples_b200 import engine  # noqa: E402
from retinanet_examples_b200.model import Model, make_state_dict  # noqa: E402


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--classes", type=int, default=80)
    ap.add_argument("--scope", choices=("heads", "fpn"), default="heads")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    dev = "cuda:0"
    g = torch.Generator().manual_seed(0)
    m = Model("ResNet50FPN", classes=args.classes).load_state_dict(make_state_dict("ResNet50FPN", args.classes, 9, False)).cuda(0)
    m.set_train_scope(args.scope)
    opt = torch.optim.SGD(m.parameters(), lr=1e-4, weight_decay=1e-4, momentum=0.9)
    scaler = torch.amp.GradScaler("cuda")
    x = torch.randn((args.batch, 3, 800, 1280), generator=g).to(dev)
    t = torch.full((args.batch, 8, 5), -1.0)
    for i in range(args.batch):
        for k in range(6):
            t[i, k] = torch.tensor([100.0 * k + 20, 60.0 * k + 30, 150.0, 120.0, float(k % args.classes)])
    t = t.to(dev)
    m.train()

    def step(split=None):
        opt.zero_grad()
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        e[0].record()
        cls_loss, box_loss = m([x, t])
        e[1].record()
        scaler.scale(cls_loss + box_loss).backward()
        e[2].record()
        scaler.step(opt)
        scaler.update()
        if split is not None:
            torch.cuda.synchronize()
            split.append((e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2])))

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    step_ms = timed(step, args.steps)
    split = []
    for _ in range(args.steps):
        step(split)
    fwd_loss = sum(s[0] for s in split) / len(split)
    bwd = sum(s[1] for s in split) / len(split)
    # the loss alone, on the head outputs of the last training forward
    m.want_atlas_grad = True
    m([x, t])
    st = m.last_train
    m.want_atlas_grad = False
    loss_ms = timed(lambda: m._compute_loss(x, st["heads"]["cls_head"], st["heads"]["box_head"], t, with_grad=True), args.steps)
    # one tower layer over the atlas: forward, weight gradient, masked input gradient
    at, P = st["at"], m._packed
    a0, a1 = at["buf"][0], at["train"]["cls_head"][0]
    gbuf = torch.zeros_like(a0)
    gin = (torch.randn(a0.shape, generator=g) * 0.01).half().to(dev) * (a1 > 0)
    conv = P["cls_head"][1]
    wd = engine.pack_weight_dgrad(dict(m.named_parameters())["cls_head.2.weight"], 256)
    launches = {
        "tower_forward": lambda: engine.conv2d(a1, conv.w, conv.b, 256, 3, relu=True, out=gbuf, tile_tab=at["tab"]),
        "tower_wgrad": lambda: engine.conv_wgrad(gin, a1, 256, tile_tab=at["tab"]),
        "tower_dgrad": lambda: engine.conv2d_dgrad(gin, wd, 256, mask=a1, tile_tab=at["tab"], out=gbuf),
    }
    flops = 2 * at["px"] * 256 * 9 * 256
    per_launch = {}
    for k, fn in launches.items():
        fn()
        ms = timed(fn, 20)
        per_launch[k] = {"ms": round(ms, 4), "tflops": round(flops / ms / 1e9, 1)}
    head_bwd = None
    if args.scope == "fpn":
        params = dict(m.named_parameters())
        fpn = m._fpn_param_names()
        for k in fpn:                     # the heads' share: the same backward with d(atlas) but no FPN gradient
            params[k].requires_grad_(False)
        m.want_atlas_grad = True
        split_h = []
        for _ in range(args.steps):
            step(split_h)
        m.want_atlas_grad = False
        for k in fpn:
            params[k].requires_grad_(True)
        head_bwd = sum(s[1] for s in split_h) / len(split_h)
        S, views = st["fpn"], st["views"]
        rows, tabs = at["rows"], at["tabs"]
        ga = (torch.randn(a0.shape, generator=g) * 0.01).half().to(dev)
        p5v = engine.AtlasView(gbuf, rows[2], views[2].h, views[2].w)
        # layer: (input, ksize, stride, level, forward launch)
        layers = {
            "lateral3": (S["c3"], 1, 1, 0, lambda: P["lateral3"](S["c3"], upsample=S["p4"])),
            "lateral4": (S["c4"], 1, 1, 1, lambda: P["lateral4"](S["c4"], upsample=S["p5"])),
            "lateral5": (S["c5"], 1, 1, 2, lambda: P["lateral5"](S["c5"])),
            "smooth3": (S["p3"], 3, 1, 0, lambda: P["smooth3"](S["p3"], out=engine.AtlasView(gbuf, rows[0], views[0].h, views[0].w))),
            "smooth4": (S["p4"], 3, 1, 1, lambda: P["smooth4"](S["p4"], out=engine.AtlasView(gbuf, rows[1], views[1].h, views[1].w))),
            "smooth5": (S["p5"], 3, 1, 2, lambda: P["smooth5"](S["p5"], out=p5v)),
            "pyramid6": (S["c5"], 3, 2, 3, lambda: P["pyramid6"](S["c5"], out=engine.AtlasView(gbuf, rows[3], views[3].h, views[3].w))),
            "pyramid7": (S["r6"], 3, 2, 4, lambda: P["pyramid7"](S["r6"], out=engine.AtlasView(gbuf, rows[4], views[4].h, views[4].w))),
        }
        for name, (xin, ks, stride, l, fwd) in layers.items():
            fl = 2 * args.batch * views[l].h * views[l].w * 256 * ks * ks * xin.shape[3]
            wg = lambda: engine.conv_wgrad_ex(ga, xin, 256, ks, stride, tabs[l], rows[l])   # noqa: E731
            for key, fn in (("forward", fwd), ("wgrad", wg)):
                fn()
                ms = timed(fn, 20)
                per_launch["%s_%s" % (name, key)] = {"ms": round(ms, 4), "tflops": round(fl / ms / 1e9, 1)}
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        gpu = torch.cuda.get_device_name(0)
    out = {"workload": "ResNet50FPN heads training, %d x 3x800x1280, %d classes" % (args.batch, args.classes),
           "gpu": gpu, "step_ms": round(step_ms, 3), "forward_ms": round(fwd_loss - loss_ms, 3),
           "loss_ms": round(loss_ms, 3), "backward_ms": round(bwd, 3), "tower_launches": per_launch,
           "tower_layer_gflop": round(flops / 1e9, 1)}
    if head_bwd is not None:
        out["workload"] = out["workload"].replace("heads training", "FPN + heads training")
        out["head_backward_ms"] = round(head_bwd, 3)
        out["fpn_backward_ms"] = round(bwd - head_bwd, 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
