"""Full precision (Model.set_precision("fp32")) vs fp16 on the flagship workload: ResNet50FPN, batch 32, 3 x 800 x 1280, class
head calibrated on the CPU oracle exactly as bench.py's FullWorkload does.

Reports, as one JSON line:
  * img/s of the fp16 and the fp32 CUDA graphs, timed in the same process, alternating, CUDA events around `--steps`
    steps after warm-up (median of `--reps` windows each);
  * per-launch times of every fp32 convolution of one eager, single-stream forward (odtk_prof_get_list), with the
    algorithmic TFLOP/s (2 * pixels * Cout * taps * Cin per time) and the tensor TFLOP/s (three tf32 MMAs per product)
    against the 495 TFLOP/s dense TF32 data-sheet peak of the H100 SXM; grouped by stage, plus the full list;
  * the fp32 vs fp16 detection match rate (same class, every box coordinate within 2 px, score within 0.02);
  * the fp32 heads' max error (per tensor, relative to max|ref|) on one image against the fp32 CPU oracle
    (oracle/model_ref.py) and against the same oracle run in float64, the fp16 heads' error against float64, and the
    fp32 oracle's own distance from float64 -- which of them is the floor;
  * the card name and power limit (read-only nvidia-smi query)."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import model_ref  # noqa: E402
from retinanet_examples_b200 import _lib, engine, synth  # noqa: E402
from retinanet_examples_b200.model import RESNET_LAYERS, Model, make_state_dict  # noqa: E402

PEAK_TF32 = 495.0            # H100 SXM dense TF32 tensor TFLOP/s (data sheet)
F32_KINDS = ("conv1x1_f32", "conv3x3_f32", "stem7x7_f32")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")[:2]]
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": "unknown (%s)" % type(e).__name__}


def launch_names(backbone):
    """Names of the fp32 convolution launches of one single-stream forward, in launch order (Model._stem, Model._features and
    the atlas heads: the class tower and its 5 final launches first, then the box tower)."""
    block, layers = RESNET_LAYERS[backbone]
    out = ["stem"]
    for li, nb in enumerate(layers):
        for b in range(nb):
            p = "layer%d.%d." % (li + 1, b)
            down = b == 0 and (li > 0 or block == "bottleneck")
            out += ([p + "downsample"] if down else []) + [p + "conv%d" % k for k in range(1, 4 if block == "bottleneck" else 3)]
    out += ["lateral5", "lateral4", "lateral3", "smooth3", "smooth4", "smooth5", "pyramid6", "pyramid7"]
    for head in ("cls_head", "box_head"):
        out += ["%s.%d" % (head, i) for i in (0, 2, 4, 6)] + ["%s.8.P%d" % (head, l) for l in range(3, 8)]
    return out


def group_of(name):
    if name.startswith(("cls_head.8", "box_head.8")):
        return name[:10]
    if name.startswith(("cls_head", "box_head")):
        return "head_towers"
    if name.startswith("layer"):
        return name.split(".")[0]
    return "stem" if name == "stem" else "fpn"


def f32_launches(model, x, backbone):
    """Per-launch ms and trace entry of every fp32 convolution of one eager, single-stream forward."""
    lib = _lib.lib()
    model.parallel_heads = False
    engine.STATS["trace"] = []
    lib.odtk_prof_reset()
    lib.odtk_prof_enable(1)
    model.forward(x)
    torch.cuda.synchronize()
    lib.odtk_prof_enable(0)
    trace, engine.STATS["trace"] = engine.STATS["trace"], None
    model.parallel_heads = True
    convs = [t for t in trace if t["kind"] in F32_KINDS]
    buf = (ctypes.c_float * len(convs))()
    assert lib.odtk_prof_get_list(3, buf, len(convs)) == len(convs)
    names = launch_names(backbone)
    assert len(names) == len(convs), (len(names), len(convs))
    rows = []
    for n, t, ms in zip(names, convs, buf):
        ms = float(ms)
        alg = t["flops"] / ms / 1e9
        rows.append({"layer": n, "shape": "%dx%dx%d %d->%d k%d s%d" % (t["n"], t["h"], t["w"], t["cin"], t["cout"],
                                                                        3 if "3x3" in t["kind"] else 7 if "stem" in t["kind"] else 1,
                                                                        t.get("stride", 1)),
                     "us": round(ms * 1e3, 1), "gflop": round(t["flops"] / 1e9, 2), "alg_tflops": round(alg, 1),
                     "tensor_tflops": round(3 * alg, 1), "tensor_share_of_495": round(3 * alg / PEAK_TF32, 3)})
    return rows


def groups(rows):
    out = {}
    for r in rows:
        g = out.setdefault(group_of(r["layer"]), {"launches": 0, "us": 0.0, "gflop": 0.0})
        g["launches"] += 1
        g["us"] += r["us"]
        g["gflop"] += r["gflop"]
    for g in out.values():
        alg = g["gflop"] / g["us"] * 1e3
        g["us"], g["gflop"] = round(g["us"], 1), round(g["gflop"], 1)
        g["alg_tflops"], g["tensor_tflops"] = round(alg, 1), round(3 * alg, 1)
        g["tensor_share_of_495"] = round(3 * alg / PEAK_TF32, 3)
    return out


def match_rate(got, ref, score_tol=0.02, px=2.0):
    hit = n = 0
    for img in range(ref[0].shape[0]):
        gs, gb, gc = [t[img] for t in got]
        rs, rb, rc = [t[img] for t in ref]
        k = int((rs > 0).sum())
        for i in range(k):
            ok = (gc == rc[i]) & (np.abs(gb - rb[i]).max(axis=1) <= px) & (np.abs(gs - rs[i]) <= score_tol)
            hit += bool(ok.any())
        n += k
    return hit / max(n, 1), n


def heads_f64(sd, backbone, x):
    """model_ref's heads (logits) in float64: its building blocks on float64 weights and input."""
    sd64 = {k: v.double() for k, v in sd.items()}
    with torch.no_grad():
        feats = model_ref.features(sd64, backbone, x.double(), False)
        return [model_ref.head(sd64, h, t) for h in ("cls_head", "box_head") for t in feats]


def worst_rel(a, b):
    return max(float((u.double().cpu() - v.double()).abs().max() / v.double().abs().max()) for u, v in zip(a, b))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-oracle", action="store_true", help="leave out the CPU oracle comparison (minutes of CPU time)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fp32_bench.py measures on a GPU; none is visible")
    dev = torch.device("cuda", 0)
    backbone, H, W = "ResNet50FPN", 800, 1280
    sd = make_state_dict(backbone, 80, 9, False, seed=0)
    probe = torch.randn((1, 3, 256, 384), generator=torch.Generator().manual_seed(3))
    sd = synth.calibrate_cls_head(sd, lambda s: model_ref.forward_heads(s, backbone, probe, sigmoid=False)[0])
    x = torch.randn((args.batch, 3, H, W), generator=torch.Generator().manual_seed(1000)).to(dev)
    models = {"fp16": Model(backbone, classes=80).load_state_dict(sd).cuda(0),
              "fp32": Model(backbone, classes=80).load_state_dict(sd).cuda(0).set_precision("fp32")}

    rows = f32_launches(models["fp32"], x, backbone)
    outs = {p: [t.clone().cpu().numpy() for t in m.forward(x)] for p, m in models.items()}
    rate, ndet = match_rate(outs["fp32"], outs["fp16"])
    res = {"workload": "%s batch %d 3x%dx%d, fp16 vs fp32 (split-TF32)" % (backbone, args.batch, H, W)}
    res.update(gpu_info())
    if not args.skip_oracle:
        x1 = x[:1].cpu()
        ref32 = [t for h in model_ref.forward_heads(sd, backbone, x1, sigmoid=False) for t in h]
        ref64 = heads_f64(sd, backbone, x1)
        got = {p: [t for h in m.forward_heads(x[:1], sigmoid=False) for t in h] for p, m in models.items()}
        res["heads_max_rel_err_1_image"] = {
            "fp32_vs_fp32_oracle": worst_rel(got["fp32"], ref32), "fp32_vs_float64_oracle": worst_rel(got["fp32"], ref64),
            "fp16_vs_float64_oracle": worst_rel(got["fp16"], ref64), "fp32_oracle_vs_float64_oracle": worst_rel(ref32, ref64)}

    for m in models.values():
        m.enable_cuda_graph()
        for _ in range(args.warmup):
            m(x)
    torch.cuda.synchronize()
    windows = {p: [] for p in models}
    for _ in range(args.reps):
        for p, m in models.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(args.steps):
                m(x)
            t1.record()
            t1.synchronize()
            windows[p].append(t0.elapsed_time(t1))
    for p in models:
        ms = float(np.median(windows[p])) / args.steps
        res["%s_img_s" % p] = round(args.batch * 1000.0 / ms, 1)
        res["%s_ms_per_step" % p] = round(ms, 3)
    res["fp32_vs_fp16_throughput"] = round(res["fp32_img_s"] / res["fp16_img_s"], 3)
    res["match_rate_fp32_vs_fp16"] = round(rate, 4)
    res["detections_compared"] = ndet
    tot_us = sum(r["us"] for r in rows)
    tot_gf = sum(r["gflop"] for r in rows)
    res["fp32_convs"] = {"launches": len(rows), "ms": round(tot_us / 1e3, 3), "alg_tflops": round(tot_gf / tot_us * 1e3, 1),
                         "tensor_tflops": round(3 * tot_gf / tot_us * 1e3, 1),
                         "tensor_share_of_495": round(3 * tot_gf / tot_us * 1e3 / PEAK_TF32, 3),
                         "groups": groups(rows), "per_launch": rows}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
