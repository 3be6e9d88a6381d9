"""INT8 vs fp16 heads on the flagship workload: ResNet50FPN, batch 32, 3 x 800 x 1280, class head calibrated on the CPU
oracle exactly as bench.py's FullWorkload does.  The INT8 model is calibrated (entropy) on a few seeded synthetic batches.

Reports, as one JSON line:
  * img/s of the fp16 and the INT8 CUDA graphs, timed in the same process, alternating, CUDA events around `--steps`
    steps after warm-up (median of `--reps` windows each);
  * per-launch times of the 8 head-tower and 10 final-layer convolutions in each precision (odtk_prof_get_list over one
    eager pass) and the achieved TOPS against the H100 SXM data-sheet dense peaks (989 fp16, 1979 INT8);
  * the quantise launch of the INT8 path;
  * the INT8 vs fp16 detection match rate (same class, every box coordinate within 2 px, score within 0.02);
  * the card name and power limit (read-only nvidia-smi query).
--scope network adds a third arm, INT8 network scope (ResNet layer3, layer4 and the FPN on s8 too), and reports:
  * fp16, INT8-heads and INT8-network img/s from CUDA graphs timed in the same process, alternating;
  * per-launch times of the layer3 / layer4 / FPN convolutions in fp16 and in INT8-network, with achieved TOPS against the
    989 / 1979 data-sheet peaks;
  * the C3 quantise launch (CUDA events over repeated launches on a C3-shaped tensor);
  * the INT8-network vs fp16 detection match rate.
--dump-outputs DIR writes every arm's detections as float32 .npy."""
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

PEAK_TOPS = {"fp16": 989.0, "int8": 1979.0}
CONV_KINDS = ("conv1x1", "conv3x3", "stem7x7", "stem_pool", "bneck_tail", "conv1x1_s8", "conv3x3_s8")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")[:2]]
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": "unknown (%s)" % type(e).__name__}


def head_launches(model, x):
    """Per-launch ms, FLOPs and kind of the 18 head convolutions of one eager, single-stream forward (the last 18 launches
    tagged conv; the quantise launch of the INT8 path is tagged as a small layer)."""
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
    convs = [t for t in trace if t["kind"] in CONV_KINDS]
    buf = (ctypes.c_float * len(convs))()
    n = lib.odtk_prof_get_list(3, buf, len(convs))
    assert n == len(convs), (n, len(convs))
    heads = list(zip(convs, buf))[-18:]
    q = [t for t in trace if t["kind"] == "quantize_s8"]
    qms = None
    if q:
        lbuf = (ctypes.c_float * 64)()
        k = lib.odtk_prof_get_list(5, lbuf, 64)
        qms = float(lbuf[k - 1])            # the quantise launch is the last small-layer launch before the heads
    return heads, qms


def region_launches(model, x, names):
    """Per-launch ms and trace entry of the layer3 / layer4 / FPN convolutions (`names`, forward order) of one eager,
    single-stream forward: the len(names) convolution launches before the 18 head convolutions."""
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
    convs = [t for t in trace if t["kind"] in CONV_KINDS]
    buf = (ctypes.c_float * len(convs))()
    assert lib.odtk_prof_get_list(3, buf, len(convs)) == len(convs)
    rows = list(zip(convs, buf))[-18 - len(names):-18]
    return [{"layer": n, "kind": t["kind"], "ms": float(v), "flops": t["flops"]} for n, (t, v) in zip(names, rows)]


def region_names(backbone):
    """The convolutions of layer3, layer4 and the FPN in launch order (downsample first in a block's first launch)."""
    block, layers = RESNET_LAYERS[backbone]
    f, out = "layer", []
    for li in (3, 4):
        for b in range(layers[li - 1]):
            p = "%s%d.%d." % (f, li, b)
            out += ([p + "downsample"] if b == 0 else []) + [p + "conv%d" % k for k in range(1, 4 if block == "bottleneck" else 3)]
    return out + ["lateral5", "lateral4", "lateral3", "smooth3", "smooth4", "smooth5", "pyramid6", "pyramid7"]


def region_table(rows16, rows8):
    table = []
    for a, b in zip(rows16, rows8):
        assert a["layer"] == b["layer"] and a["flops"] == b["flops"], (a, b)
        table.append({"layer": a["layer"], "gflop": round(a["flops"] / 1e9, 2),
                      "fp16_us": round(a["ms"] * 1e3, 1), "fp16_tops": round(a["flops"] / a["ms"] / 1e9, 1),
                      "int8_us": round(b["ms"] * 1e3, 1), "int8_tops": round(b["flops"] / b["ms"] / 1e9, 1),
                      "speedup": round(a["ms"] / b["ms"], 2)})
    tot16, tot8 = sum(r["ms"] for r in rows16), sum(r["ms"] for r in rows8)
    fl = sum(r["flops"] for r in rows16)
    return {"launches": table, "fp16_ms": round(tot16, 3), "int8_ms": round(tot8, 3),
            "fp16_share_of_peak": round(fl / tot16 / 1e9 / PEAK_TOPS["fp16"], 3),
            "int8_share_of_peak": round(fl / tot8 / 1e9 / PEAK_TOPS["int8"], 3)}


def quantize_ms(c3_shape, dev, reps=50):
    """One C3 quantise launch (odtk_quantize_f16_s8), CUDA events over `reps` launches after a warm-up."""
    t = torch.randn(c3_shape, generator=torch.Generator().manual_seed(7)).half().to(dev)
    out = torch.empty(c3_shape, dtype=torch.int8, device=dev)
    for _ in range(5):
        engine.quantize_f16_s8(t, 10.0, out=out)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        engine.quantize_f16_s8(t, 10.0, out=out)
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / reps


def summarize(heads, precision):
    groups = {"tower": heads[0:4] + heads[9:13], "cls_final": heads[4:9], "box_final": heads[13:18]}
    out = {}
    for g, rows in groups.items():
        ms = sum(float(v) for _, v in rows)
        fl = sum(t["flops"] for t, _ in rows)
        out[g] = {"launches": len(rows), "ms": round(ms, 4), "tops": round(fl / ms / 1e9, 1),
                  "share_of_peak": round(fl / ms / 1e9 / PEAK_TOPS[precision], 3),
                  "per_launch_us": [round(float(v) * 1e3, 1) for _, v in rows]}
    ms = sum(float(v) for _, v in heads)
    fl = sum(t["flops"] for t, _ in heads)
    out["all_heads"] = {"ms": round(ms, 4), "tops": round(fl / ms / 1e9, 1), "share_of_peak": round(fl / ms / 1e9 / PEAK_TOPS[precision], 3)}
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--calib-batches", type=int, default=2)
    ap.add_argument("--calib-batch-size", type=int, default=8)
    ap.add_argument("--method", default="entropy", choices=("entropy", "max"))
    ap.add_argument("--scope", default="heads", choices=("heads", "network"))
    ap.add_argument("--dump-outputs", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("int8_bench.py measures on a GPU; none is visible")
    dev = torch.device("cuda", 0)
    backbone, H, W = "ResNet50FPN", 800, 1280
    sd = make_state_dict(backbone, 80, 9, False, seed=0)
    probe = torch.randn((1, 3, 256, 384), generator=torch.Generator().manual_seed(3))
    sd = synth.calibrate_cls_head(sd, lambda s: model_ref.forward_heads(s, backbone, probe, sigmoid=False)[0])
    x = torch.randn((args.batch, 3, H, W), generator=torch.Generator().manual_seed(1000)).to(torch.float16) \
        .contiguous(memory_format=torch.channels_last).to(dev)
    m16 = Model(backbone, classes=80).load_state_dict(sd).cuda(0)
    m8 = Model(backbone, classes=80).load_state_dict(sd).cuda(0)
    calib_x = [torch.randn((args.calib_batch_size, 3, H, W), generator=torch.Generator().manual_seed(2000 + i))
               for i in range(args.calib_batches)]
    table = m8.calibrate(calib_x, method=args.method, scope=args.scope)
    m8.set_precision("int8", table)
    models = {"fp16": m16, "int8": m8}
    if args.scope == "network":
        mn = Model(backbone, classes=80).load_state_dict(sd).cuda(0)
        mn.set_precision("int8", table, scope="network")
        models["int8_network"] = mn

    heads = {p: head_launches(m, x) for p, m in models.items() if p != "int8_network"}
    outs = {p: [t.clone().cpu().numpy() for t in m.forward(x)] for p, m in models.items()}
    rate, ndet = match_rate(outs["int8"], outs["fp16"])
    if args.scope == "network":
        names = region_names(backbone)
        region = region_table(region_launches(m16, x, names), region_launches(models["int8_network"], x, names))
        rate_net, _ = match_rate(outs["int8_network"], outs["fp16"])
    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        for p, o in outs.items():
            for name, t in zip(("scores", "boxes", "classes"), o):
                np.save(os.path.join(args.dump_outputs, "%s_%s.npy" % (p, name)), t.astype(np.float32))

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
    res = {"workload": "%s batch %d 3x%dx%d, %s (%s calibration, %d x %d images)" % (
        backbone, args.batch, H, W, "heads fp16 vs INT8" if args.scope == "heads" else "fp16 vs INT8 heads vs INT8 network",
        args.method, args.calib_batches, args.calib_batch_size)}
    res.update(gpu_info())
    for p in models:
        ms = float(np.median(windows[p])) / args.steps
        res["%s_img_s" % p] = round(args.batch * 1000.0 / ms, 1)
        res["%s_ms_per_step" % p] = round(ms, 3)
        if p in heads:
            res["%s_heads" % p] = summarize(heads[p][0], p)
    res["int8_speedup"] = round(res["int8_img_s"] / res["fp16_img_s"], 3)
    res["int8_quantize_ms"] = round(heads["int8"][1], 4) if heads["int8"][1] is not None else None
    res["match_rate_int8_vs_fp16"] = round(rate, 4)
    res["detections_compared"] = ndet
    if args.scope == "network":
        res["int8_network_speedup"] = round(res["int8_network_img_s"] / res["fp16_img_s"], 3)
        res["int8_network_vs_heads"] = round(res["int8_network_img_s"] / res["int8_img_s"], 3)
        res["layer3_layer4_fpn"] = region
        res["c3_quantize_ms"] = round(quantize_ms((args.batch, H // 8, W // 8, 512), dev), 4)
        res["match_rate_int8_network_vs_fp16"] = round(rate_net, 4)
    res["scales"] = table["scales"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
