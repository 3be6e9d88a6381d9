"""Raw-image input side (odtk_preprocess_resize_u8 / Model.forward_images) on one GPU; prints one JSON line.

    python tools/preprocess_bench.py [--batch 32] [--steps 20] [--warmup 5]

Inputs: a seeded mix of COCO-like image sizes (640 x 480, 427 x 640, 500 x 375, ...), resize 800, max_size 1333 (the
reference's defaults), one canvas: the mix's reference collate.  Reports
  * kernel: odtk_preprocess_resize_u8 alone over the staged batch, CUDA events: us per image, algorithmic bytes (every
    source byte and the size table read once, the whole fp16 NHWC4 canvas written once) over time in GB/s and as a share
    of the H100 SXM data-sheet 3.35 TB/s;
  * cpu_reference: the reference's per-image CPU work on one thread (PIL BILINEAR resize, then torch normalise and pad as
    odtk/data.py:113-123 does), ms per image, and the host's core count;
  * e2e: ResNet50FPN img/s at this batch, CUDA graphs, alternating two arms in one process: forward_images from pinned
    host uint8 lists (upload + resize + network) against model(x) on a prebuilt fp32 device batch of the same canvas
    holding the same pixels (network only); the two arms' detections are compared;
  * the card name and power limit (read-only nvidia-smi query)."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from retinanet_examples_b200 import engine  # noqa: E402
from retinanet_examples_b200.model import Model, make_state_dict  # noqa: E402

COCO_SIZES = [(480, 640), (427, 640), (640, 480), (640, 427), (375, 500), (500, 375), (612, 612), (360, 640), (424, 640),
              (480, 640), (640, 640), (333, 500)]
HBM_GBS = 3350.0


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")[:2]]
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": "unknown (%s)" % type(e).__name__}


def images(batch, seed=0):
    rng = np.random.default_rng(seed)
    shapes = [COCO_SIZES[int(i)] for i in rng.integers(0, len(COCO_SIZES), batch)]
    return [torch.from_numpy(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)) for h, w in shapes]


def time_events(fn, steps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / steps


def kernel_arm(imgs, steps, warmup):
    plan = engine.ResizePlan([i.shape[:2] for i in imgs], 800, 1333)
    buf = torch.empty(engine.table_pad(plan.n) + plan.nbytes, dtype=torch.uint8, device="cuda")
    tab, x = engine.stage_images(imgs, plan, buf)
    out = engine.resize_launch(x, plan.nbytes, plan, tab)
    for _ in range(warmup):
        engine.resize_launch(x, plan.nbytes, plan, tab, out=out)
    ms = min(time_events(lambda: engine.resize_launch(x, plan.nbytes, plan, tab, out=out), steps) for _ in range(3))
    nbytes = engine.resize_bytes(plan)
    return {"canvas": list(plan.canvas), "us_per_image": ms * 1e3 / plan.n, "ms_per_batch": ms, "bytes": nbytes,
            "GBps": nbytes / ms / 1e6, "share_of_3350GBps": nbytes / ms / 1e6 / HBM_GBS}


def cpu_reference_arm(imgs, count):
    """odtk/data.py:55-60 and 113-123 on one thread: PIL resize, ByteTensor -> float / 255 -> per-channel sub_ / div_ ->
    stride pad."""
    from PIL import Image
    import torch.nn.functional as F
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    mean, std, stride = engine.IMAGENET_MEAN, engine.IMAGENET_STD, 128
    pil = [Image.fromarray(i.numpy(), "RGB") for i in imgs[:count]]
    t0 = time.perf_counter()
    for im in pil:
        ratio = 800 / min(im.size)
        if ratio * max(im.size) > 1333:
            ratio = 1333 / max(im.size)
        im = im.resize(tuple(int(ratio * d) for d in im.size), Image.BILINEAR)
        data = torch.ByteTensor(torch.ByteStorage.from_buffer(im.tobytes()))
        data = data.float().div(255).view(*im.size[::-1], len(im.mode)).permute(2, 0, 1)
        for t, m, s in zip(data, mean, std):
            t.sub_(m).div_(s)
        pw, ph = ((stride - d % stride) % stride for d in im.size)
        F.pad(data, (0, pw, 0, ph))
    ms = (time.perf_counter() - t0) * 1e3 / len(pil)
    torch.set_num_threads(threads)
    return {"ms_per_image_one_thread": ms, "images": len(pil), "host_cores": os.cpu_count()}


def e2e_arm(imgs, steps, warmup, rounds=3):
    sd = make_state_dict("ResNet50FPN", 80, 9, False, seed=0)
    m = Model("ResNet50FPN", classes=80).load_state_dict(sd).cuda()
    pinned = [i.pin_memory() for i in imgs]
    xp, hs, ws, _ = engine.preprocess_resize_u8(imgs, 800, 1333)
    x = xp[:, 3:3 + hs, 3:3 + ws, :3].permute(0, 3, 1, 2).float().contiguous()        # the same pixels, prebuilt
    m.enable_cuda_graph()
    arms = {"forward_images": lambda: m.forward_images(pinned, 800, 1333, (hs, ws)),
            "model_x_prebuilt": lambda: m(x, static_input=True)}
    outs = {}
    for k, fn in arms.items():
        for _ in range(warmup):
            fn()
        outs[k] = [t.clone() for t in (fn()[0] if k == "forward_images" else fn())]
    torch.cuda.synchronize()
    res = {k: [] for k in arms}
    for _ in range(rounds):                   # alternate the arms; host clock around work that ends in a synchronise
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                fn()
            torch.cuda.synchronize()
            res[k].append(len(imgs) * steps / (time.perf_counter() - t0))
    same = all(torch.equal(a, b) for a, b in zip(outs["forward_images"], outs["model_x_prebuilt"]))
    return {"canvas": [hs, ws], "img_per_s": {k: float(np.median(v)) for k, v in res.items()},
            "img_per_s_rounds": res, "detections_identical": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--cpu-images", type=int, default=32)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("preprocess_bench needs a CUDA device")
    imgs = images(a.batch)
    res = {"bench": "preprocess_resize_u8", "batch": a.batch, "resize": 800, "max_size": 1333, **card()}
    res["kernel"] = kernel_arm(imgs, a.steps * 5, a.warmup)
    res["cpu_reference"] = cpu_reference_arm(imgs, a.cpu_images)
    res["e2e_resnet50fpn"] = e2e_arm(imgs, a.steps, a.warmup)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
