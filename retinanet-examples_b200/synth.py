"""Deterministic synthetic workloads of the shapes BASELINE.json names.
No dataset or checkpoint exists offline: head outputs follow the measured candidate statistics
(cls logits ~ N(-7, 1.6^2) -> ~0.56 % of scores above 0.05; box deltas ~ N(0, 0.2^2))."""
import math

import torch

LEVEL_STRIDES = (8, 16, 32, 64, 128)


def level_sizes(height=800, width=1280):
    """Feature-map sizes of P3..P7 for an input of height x width (3x3 s2 p1 convs after C5)."""
    sizes = []
    h, w = height, width
    for _ in range(3):      # stem s2, maxpool s2, layer2 s2  -> stride 8
        h, w = (h + 1) // 2, (w + 1) // 2
    for _ in range(5):
        sizes.append((h, w))
        h, w = (h + 1) // 2, (w + 1) // 2
    return sizes


def head_outputs(batch, height=800, width=1280, classes=80, anchors=9, rotated=False, seed=0,
                 device="cpu", mean=-7.0, std=1.6, dtype=torch.float32):
    """Returns per-level lists (scores [B, A*C, H, W] after sigmoid, deltas [B, A*4|6, H, W])."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    nbox = 6 if rotated else 4
    cls, box = [], []
    for (h, w) in level_sizes(height, width):
        z = torch.randn((batch, anchors * classes, h, w), generator=g) * std + mean
        s = torch.sigmoid(z).to(dtype)
        d = torch.randn((batch, anchors * nbox, h, w), generator=g) * 0.2
        if rotated:  # sin/cos channels: theta ~ U(-pi/4, pi/4)
            theta = (torch.rand((batch, anchors, h, w), generator=g) - 0.5) * (math.pi / 2)
            d = d.view(batch, anchors, 6, h, w)
            d[:, :, 4] = torch.sin(theta)
            d[:, :, 5] = torch.cos(theta)
            d = d.view(batch, anchors * 6, h, w)
        cls.append(s.to(device))
        box.append(d.to(dtype).to(device))
    return cls, box


def calibrate_cls_head(sd, logits_fn, mean=-7.0, std=1.6, seed=0):
    """Rescale the last class-head convolution of a random-init state_dict so that its logits follow
    ~N(mean, std^2) (~0.56 % of scores above 0.05, so decode and NMS do
    representative work; a fresh model yields zero detections).  `logits_fn(state_dict)` must return
    the per-level raw class logits of some probe batch under these weights (the caller decides
    how: the GPU engine via Model.forward_heads(sigmoid=False) in the product arm)."""
    g = torch.Generator().manual_seed(seed)
    w8 = torch.randn(sd["cls_head.8.weight"].shape, generator=g) * 0.01
    sd = dict(sd)
    sd["cls_head.8.weight"], sd["cls_head.8.bias"] = w8, torch.zeros_like(sd["cls_head.8.bias"])
    flat = torch.cat([l.float().reshape(-1).cpu() for l in logits_fn(sd)])
    s = std / float(flat.std())
    sd["cls_head.8.weight"] = w8 * s
    sd["cls_head.8.bias"] = torch.full_like(sd["cls_head.8.bias"], mean - s * float(flat.mean()))
    return sd
