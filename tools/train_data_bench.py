"""Training input path (retinanet_examples_b200.data.DataIterator) on one GPU; prints one JSON line.

    python tools/train_data_bench.py [--batch 8] [--steps 20] [--warmup 3]

Inputs: the two 640x480 streams of tests/golden/jpeg_pil.npz (they carry restart markers every 2 MCU rows, so their GPU
entropy decode runs one thread per restart segment), and the same pixels re-encoded by Pillow without restart markers
(one entropy-decode thread per image, like typical COCO files) when Pillow is importable; synthetic annotations (three
boxes per image).  Default jitter [640, 1024], max_size 1333, default augments, rotate_augment on.  Reports per stream
set:
  * batch_ms: one iterator batch, host clock around batch() + a device synchronise, median over --steps batches;
  * host_ms: the same clock up to the return of batch() (host work and launches; the device may still be running);
  * kernels_ms: each kernel's device time from a torch.profiler run of its own (decode, resize, augment);
  * train: ResNet50FPN (heads scope, SGD + GradScaler, the reference's loop) steps per second fed by the iterator (a
    fresh batch per step, restart-marker-free streams) against the same loop on device batches prebuilt from the same
    draws (so the same canvases); host clock
    around --steps steps ending in a device synchronise, after --warmup steps of each;
  * cpu_ref_ms_per_image: Pillow decode + resize + the four torchvision colour adjustments + normalise on one host
    thread, when Pillow and torchvision are importable, else "not measured";
  * the card name and power limit (read-only nvidia-smi query)."""
import argparse
import io
import json
import os
import random
import re
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from preprocess_bench import card  # noqa: E402
from retinanet_examples_b200 import data  # noqa: E402

AUG = dict(augment_brightness=0.002, augment_contrast=0.002, augment_hue=0.0002, augment_saturation=0.002)


def stream_sets():
    g = np.load(os.path.join(ROOT, "tests", "golden", "jpeg_pil.npz"))
    sets = {"restart_markers": [g["420_640x480_jpeg"].tobytes(), g["444_480x640_jpeg"].tobytes()]}
    try:
        from PIL import Image
        plain = []
        for s in sets["restart_markers"]:
            b = io.BytesIO()
            Image.open(io.BytesIO(s)).save(b, "JPEG", quality=90)
            plain.append(b.getvalue())
        sets["no_restart_markers"] = plain
    except ImportError:
        pass
    return sets


def write_dataset(d, streams, n):
    images, anns = [], []
    for i in range(n):
        name = "im%03d.jpg" % i
        with open(os.path.join(d, name), "wb") as f:
            f.write(streams[i % len(streams)])
        images.append({"id": i + 1, "file_name": name})
        for j in range(3):
            anns.append({"id": 3 * i + j + 1, "image_id": i + 1, "category_id": 1 + j,
                         "bbox": [10.0 + 20 * j, 15.0 + 10 * j, 50.5, 40.25]})
    path = os.path.join(d, "ann.json")
    with open(path, "w") as f:
        json.dump({"images": images, "annotations": anns, "categories": [{"id": k} for k in (1, 2, 3)]}, f)
    return path


def measure(streams, batch, steps, warmup):
    with tempfile.TemporaryDirectory() as d:
        ann = write_dataset(d, streams, batch)
        it = data.DataIterator(d, [640, 1024], 1333, batch, 128, 1, ann, training=True, rotate_augment=True,
                               rng=random.Random(0), **AUG)
        idx = list(range(batch))
        for _ in range(warmup):
            it.batch(idx)
        torch.cuda.synchronize()
        total, host = [], []
        for _ in range(steps):
            t0 = time.perf_counter()
            it.batch(idx)
            t1 = time.perf_counter()
            torch.cuda.synchronize()
            total.append((time.perf_counter() - t0) * 1e3)
            host.append((t1 - t0) * 1e3)
        it._check_pending()
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                it.batch(idx)
            torch.cuda.synchronize()
        kernels = {}
        for e in prof.key_averages():
            if e.device_type == torch.autograd.DeviceType.CUDA and e.count:
                m = re.search(r"(\w+_kernel)", e.key)
                key = m.group(1) if m else e.key[:40]
                kernels[key] = round(kernels.get(key, 0.0) + e.device_time_total / 1e3 / 3, 4)
        it._check_pending()
    return {"batch_ms": round(float(np.median(total)), 3), "host_ms": round(float(np.median(host)), 3), "kernels_ms": kernels}


def train_steps(streams, batch, steps, warmup):
    from retinanet_examples_b200.model import Model, make_state_dict
    m = Model("ResNet50FPN", classes=80).load_state_dict(make_state_dict("ResNet50FPN", 80, 9, False)).cuda(0)
    m.train()
    opt = torch.optim.SGD(m.parameters(), lr=1e-4, weight_decay=1e-4, momentum=0.9)
    scaler = torch.amp.GradScaler("cuda")

    def step(data, target):
        opt.zero_grad()
        cls_loss, box_loss = m([data.contiguous(memory_format=torch.channels_last), target])
        scaler.scale(cls_loss + box_loss).backward()
        scaler.step(opt)
        scaler.update()

    out = {}
    with tempfile.TemporaryDirectory() as d:
        ann = write_dataset(d, streams, batch)
        make = lambda: data.DataIterator(d, [640, 1024], 1333, batch, 128, 1, ann, training=True,  # noqa: E731
                                         rotate_augment=True, rng=random.Random(1), **AUG)
        idx = list(range(batch))
        # both arms see the same sequence of draws, so the same canvases: the prebuilt arm's batches are made up front
        pre = make()
        fixed = [pre.batch(idx) for _ in range(warmup + steps)]
        pre._check_pending()
        it = make()
        arms = {"prebuilt_batches": lambda i: step(*fixed[i]), "iterator": lambda i: step(*it.batch(idx))}
        for name, fn in arms.items():
            for i in range(warmup):
                fn(i)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(warmup, warmup + steps):
                fn(i)
            torch.cuda.synchronize()
            out[name + "_steps_per_s"] = round(steps / (time.perf_counter() - t0), 2)
        it._check_pending()
        out["canvases"] = sorted({tuple(f[0].shape[2:]) for f in fixed})
        del fixed
    return out


def cpu_reference(streams, n=4):
    try:
        from PIL import Image
        import torchvision.transforms.functional as F
    except ImportError:
        return "not measured"
    torch.set_num_threads(1)
    rng = random.Random(0)
    t0 = time.perf_counter()
    for i in range(n):
        im = Image.open(io.BytesIO(streams[i % len(streams)])).convert("RGB")
        r = rng.randint(640, 1024) / min(im.size)
        if r * max(im.size) > 1333:
            r = 1333 / max(im.size)
        im = im.resize([int(r * s) for s in im.size], Image.BILINEAR)
        im = F.adjust_brightness(im, 1.001)
        im = F.adjust_contrast(im, 0.999)
        im = F.adjust_hue(im, 0.0001)
        im = F.adjust_saturation(im, 1.002)
        x = torch.ByteTensor(torch.ByteStorage.from_buffer(im.tobytes())).float().div(255)
        x = x.view(im.size[1], im.size[0], 3).permute(2, 0, 1)
        for t, m, s in zip(x, [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]):
            t.sub_(m).div_(s)
    return round((time.perf_counter() - t0) * 1e3 / n, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    out = {"card": card(), "batch": a.batch}
    sets = stream_sets()
    for name, streams in sets.items():
        out[name] = measure(streams, a.batch, a.steps, a.warmup)
    out["train"] = train_steps(sets.get("no_restart_markers", sets["restart_markers"]), a.batch, a.steps, a.warmup)
    out["cpu_ref_ms_per_image"] = cpu_reference(sets.get("no_restart_markers", sets["restart_markers"]))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
