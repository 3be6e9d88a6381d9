"""Time every DISTINCT layer launch of one step of bench.py's default workload in isolation (CUDA events on the
launching stream, 2 warm-up + N timed launches each) and print / save a table:
    python tools/layer_bench.py [--batch 32] [--backbone ResNet50FPN] [--reps 5] [--tag name] [--rotated] [--out DIR]
The calls are recorded by wrapping the engine's entry points while one eager forward runs, then replayed with the very
same tensors (so shapes, strides, fused epilogues and the kernel variant chosen by the host code are the model's own).
The ODTK_PDL environment toggle is read at first use: run once per setting and compare the JSON files.  Inputs of the small pyramid levels fit the L2, exactly as they do inside the real step."""
import argparse
import collections
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--backbone", default="ResNet50FPN")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--tag", default="base")
    ap.add_argument("--rotated", action="store_true")
    ap.add_argument("--only", default=None, help="substring filter on the layer key")
    ap.add_argument("--out", default=".", help="directory of layer_bench_<tag>.json")
    ap.add_argument("--calibrated", action="store_true", help="class-head bias calibrated like bench.py (~0.56 %% of the scores above the threshold)")
    args = ap.parse_args()
    import torch
    from retinanet_examples_b200 import engine
    from retinanet_examples_b200.model import Model, make_state_dict
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    tf, bw = 989.0, 3350.0   # H100 SXM data sheet: dense FP16 TFLOP/s, HBM3 GB/s

    calls = []
    names = ["conv2d", "stem_conv", "stem_conv_padded", "maxpool3x3s2", "lower_conv", "relu", "pad_input", "stem_pool_padded", "bottleneck_tail"]
    orig = {n: getattr(engine, n) for n in names if hasattr(engine, n)}

    def wrap(name):
        fn = orig[name]

        def inner(*a, **k):
            t0 = len(engine.STATS["trace"])
            out = fn(*a, **k)
            plan = engine.last_plan() if name in ("conv2d", "stem_conv", "stem_conv_padded") else None
            calls.append((name, a, k, engine.STATS["trace"][t0:], plan))
            return out
        return inner
    for n in orig:
        setattr(engine, n, wrap(n))

    na = 27 if args.rotated else 9
    model = Model(args.backbone, classes=80, rotated_bbox=args.rotated)
    sd = make_state_dict(args.backbone, 80, na, args.rotated, seed=0)
    if args.calibrated:
        from retinanet_examples_b200 import synth
        xp = torch.randn((2, 3, 800, 1280), generator=torch.Generator().manual_seed(1)).to(torch.float16).contiguous(memory_format=torch.channels_last).to(dev)

        def gpu_logits(s):
            engine.STATS["trace"] = []
            model.load_state_dict(s).cuda(0)
            return model.forward_heads(xp, sigmoid=False)[0]
        sd = synth.calibrate_cls_head(sd, gpu_logits)
    model.load_state_dict(sd).cuda(0)
    model.parallel_heads = False
    x = torch.randn((args.batch, 3, 800, 1280), generator=torch.Generator().manual_seed(1)).to(torch.float16) \
        .contiguous(memory_format=torch.channels_last).to(dev)
    with torch.no_grad():
        engine.STATS["trace"] = []
        model.forward(x)                      # warm-up (lazy init)
        calls.clear()
        engine.STATS["trace"] = []
        model.forward(x)
    torch.cuda.synchronize()
    for n in orig:
        setattr(engine, n, orig[n])
    engine.STATS["trace"] = None

    def key(tr):
        return " + ".join("%s %dx%dx%d %s->%s%s%s%s%s" % (
            t["kind"], t["n"], t["h"], t["w"], t["cin"], t.get("cout", ""), " s2" if t.get("stride") == 2 else "",
            " +res" if t.get("residual") else "", " +up" if t.get("upsample") else "",
            {1: " f32", 2: " f32sig", 3: " cand"}.get(t.get("out_mode"), "")) for t in tr)

    groups = collections.OrderedDict()
    for c in calls:
        g = groups.setdefault(key(c[3]), {"n": 0, "call": c})
        g["n"] += 1
    rows = []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.no_grad():
        for k, g in groups.items():
            if args.only and args.only not in k:
                continue
            name, a, kw, tr, plan = g["call"]
            fn = orig[name]
            sink = kw.get("sink")
            for _ in range(2):
                fn(*a, **kw)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(args.reps):
                fn(*a, **kw)
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / args.reps
            flops, byt = sum(t["flops"] for t in tr), sum(t["bytes"] for t in tr)
            ideal = max(flops / (tf * 1e12), byt / (bw * 1e9)) * 1e6
            rows.append({"layer": k, "n": g["n"], "us": round(us, 1), "ideal_us": round(ideal, 1), "eff": round(ideal / us, 3),
                         "tflops": round(flops / us / 1e6, 1), "gbs": round(byt / us / 1e3, 1), "plan": plan})
    tot = sum(r["us"] * r["n"] for r in rows)
    ideal = sum(r["ideal_us"] * r["n"] for r in rows)
    print("%-58s %3s %9s %9s %5s %8s %8s  plan" % ("layer", "n", "us", "ideal", "eff", "TFLOP/s", "GB/s"))
    for r in sorted(rows, key=lambda r: -r["us"] * r["n"]):
        p = r["plan"] or {}
        print("%-58s %3d %9.1f %9.1f %5.2f %8.1f %8.1f  %s" % (
            r["layer"][:58], r["n"], r["us"], r["ideal_us"], r["eff"], r["tflops"], r["gbs"],
            ("m%d cl%d bn%d st%d np%d t%d res%d rmma%d tmast%d up%d grid%d" % (
                p["mode"], p["cluster"], p["bn"], p["nstages"], p["npatch"], p["tile_t"], p["b_resident"], p["res_mma"],
                p["tma_store"], p["up_mma"], p["grid"])) if p else ""))
    print("sum over the step (isolated launches): %.1f us, layer-wise ideal %.1f us, frac %.3f" % (tot, ideal, ideal / tot))
    os.makedirs(args.out, exist_ok=True)
    json.dump({"tag": args.tag, "batch": args.batch, "backbone": args.backbone, "sum_us": round(tot, 1),
               "ideal_us": round(ideal, 1), "rows": rows},
              open(os.path.join(args.out, "layer_bench_%s.json" % args.tag), "w"), indent=1)


if __name__ == "__main__":
    main()
