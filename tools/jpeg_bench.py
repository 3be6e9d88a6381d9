"""GPU JPEG decode (odtk_decode_jpeg / Model.forward_jpeg) on one GPU; prints one JSON line.

    python tools/jpeg_bench.py [--batch 32] [--steps 20] [--warmup 5]

Inputs: a batch drawn from the two stored 640x480 fixtures of tests/golden/jpeg_pil.npz (4:2:0 quality 90, and 4:4:4
quality 90 with restart markers every 2 MCU rows), resize 800, max_size 1333.  Reports
  * decode: odtk_decode_jpeg over the staged batch, CUDA events over many calls: ms per batch and us per image; then a
    torch.profiler run of its own gives each kernel's time (restart scan, entropy decode, IDCT, upsample + colour);
  * e2e: ResNet50FPN img/s, CUDA graphs, alternating two arms in one process on the same canvas: forward_jpeg from the
    compressed bytes (parse, stage, decode, resize, network) against forward_images on the same images pre-decoded into
    pinned host memory (upload, resize, network); the arms' detections are compared;
  * cpu_pillow: Pillow's decode per image on one thread of this host if Pillow is installed, else "not measured";
  * the card name and power limit (read-only nvidia-smi query)."""
import argparse
import io
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from preprocess_bench import card, time_events  # noqa: E402
from retinanet_examples_b200 import engine, jpeg  # noqa: E402
from retinanet_examples_b200.model import Model, make_state_dict  # noqa: E402

STAGES = ("jpeg_restart_kernel", "jpeg_entropy_kernel", "jpeg_idct_kernel", "jpeg_color_kernel")


def streams(batch):
    g = np.load(os.path.join(ROOT, "tests", "golden", "jpeg_pil.npz"))
    both = [g["420_640x480_jpeg"].tobytes(), g["444_480x640_jpeg"].tobytes()]
    return [both[i % 2] for i in range(batch)]


def decode_arm(datas, steps, warmup):
    b = jpeg.JpegBatch(datas)
    outs, nbytes = engine._output_table(b.shapes)
    buf = b.stage(outs, torch.empty(b.nbytes, dtype=torch.uint8, device="cuda"))
    y = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    ws = torch.empty(b.workspace_bytes(), dtype=torch.uint8, device="cuda")
    st = torch.empty(b.n, dtype=torch.int32, device="cuda")
    run = lambda: engine.jpeg_launch(b, buf, outs, ws, y, st)
    for _ in range(warmup):
        run()
    ms = time_events(run, steps)
    assert st.cpu().tolist() == [0] * b.n
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            run()
        torch.cuda.synchronize()
    per = {k: 0.0 for k in STAGES}
    for e in prof.key_averages():
        for k in STAGES:
            if k in e.key:
                per[k] += e.device_time_total / 1000.0 / steps
    host_t = time.perf_counter()
    for _ in range(steps):
        jpeg.JpegBatch(datas)
    host_ms = (time.perf_counter() - host_t) * 1000 / steps
    return {"ms_per_batch": round(ms, 3), "us_per_image": round(ms * 1000 / b.n, 1),
            "stage_ms_per_batch": {k.replace("_kernel", ""): round(v, 3) for k, v in per.items()},
            "host_parse_pack_ms_per_batch": round(host_ms, 3),
            "scan_bytes_per_image": int(sum(t.scan_bytes for t in b.images) / b.n),
            "decoded_bytes_per_image": int(b.pixels * 3 / b.n), "blocks_per_image": int(b.blocks / b.n)}


def e2e_arm(datas, steps, warmup, rounds=3):
    import jpeg_oracle
    imgs = [torch.from_numpy(jpeg_oracle.decode(d)).pin_memory() for d in datas]
    sd = make_state_dict("ResNet50FPN", 80, 9, False, seed=1)
    m = Model("ResNet50FPN", classes=80).load_state_dict(sd).cuda()
    m.enable_cuda_graph()
    plan = engine.ResizePlan([tuple(i.shape[:2]) for i in imgs], 800, 1333, m.stride)
    canvas = plan.canvas
    a = lambda: m.forward_jpeg(datas, 800, 1333, canvas)
    b = lambda: m.forward_images(imgs, 800, 1333, canvas)
    got = [t.clone() for t in a()[0]]
    want = [t.clone() for t in b()[0]]
    same = all(torch.equal(u, v) for u, v in zip(got, want))
    rates = {"forward_jpeg": [], "forward_images": []}
    for _ in range(rounds):
        for name, fn in (("forward_jpeg", a), ("forward_images", b)):
            for _ in range(warmup):
                fn()
            torch.cuda.synchronize()
            t = time.perf_counter()
            for _ in range(steps):
                fn()
            torch.cuda.synchronize()
            rates[name].append(len(datas) * steps / (time.perf_counter() - t))
    return {"canvas": list(canvas), "detections_equal": same,
            **{k + "_img_s": round(float(np.median(v)), 1) for k, v in rates.items()},
            "rounds": {k: [round(x, 1) for x in v] for k, v in rates.items()}}


def cpu_pillow(datas, count=20):
    try:
        from PIL import Image
    except ImportError:
        return "not measured (Pillow is not installed on this host)"
    t = time.perf_counter()
    for i in range(count):
        np.asarray(Image.open(io.BytesIO(datas[i % 2])).convert("RGB"))
    return {"ms_per_image": round((time.perf_counter() - t) * 1000 / count, 3), "threads": 1}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--skip-e2e", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("jpeg_bench needs a CUDA device")
    datas = streams(args.batch)
    res = {"tool": "jpeg_bench", "batch": args.batch, **card(), "decode": decode_arm(datas, args.steps, args.warmup)}
    if not args.skip_e2e:
        res["e2e"] = e2e_arm(datas, args.steps, args.warmup)
    res["cpu_pillow"] = cpu_pillow(datas)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
