"""Fixture for the fused training loss: the UNMODIFIED reference Model._compute_loss
(odtk/model.py:186-210: _extract_targets -> snap_to_anchors per image and level, FocalLoss, SmoothL1Loss, masks,
foreground counts, normalisation) and its autograd gradients w.r.t. the head tensors, on seeded random heads / targets.
    python oracle/gen_golden_loss.py  ->  tests/golden/compute_loss.npz          TEST INFRASTRUCTURE ONLY."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_import  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def main():
    odtk = ref_import.import_reference()
    classes, batch, H, W = 5, 2, 128, 256
    m = odtk.model.Model("ResNet18FPN", classes=classes)
    g = torch.Generator().manual_seed(21)
    x = torch.zeros((batch, 3, H, W))
    cls_heads, box_heads = [], []
    for s in (8, 16, 32, 64, 128):
        h, w = H // s, W // s
        cls_heads.append((torch.randn((batch, 9 * classes, h, w), generator=g) * 2 - 3).requires_grad_())
        box_heads.append((torch.randn((batch, 9 * 4, h, w), generator=g) * 0.5).requires_grad_())
    rng = np.random.default_rng(4)
    t = np.full((batch, 12, 5), -1.0, np.float32)
    for b in range(batch):
        n = 9 if b == 0 else 5
        wh = rng.uniform(16, 120, size=(n, 2))
        xy = rng.uniform(0, [W - 40, H - 40], size=(n, 2))
        t[b, :n] = np.concatenate([np.round(xy), np.round(wh), rng.integers(0, classes, size=(n, 1))], 1)
    targets = torch.from_numpy(t)
    cls_loss, box_loss = m._compute_loss(x, cls_heads, box_heads, targets.float())
    (cls_loss + box_loss).backward()
    d = {"classes": classes, "targets": t, "width": W, "cls_loss": cls_loss.detach().numpy(), "box_loss": box_loss.detach().numpy()}
    for i, (c, b) in enumerate(zip(cls_heads, box_heads)):
        d["cls%d" % i], d["box%d" % i] = c.detach().numpy(), b.detach().numpy()
        d["cls_grad%d" % i], d["box_grad%d" % i] = c.grad.numpy(), b.grad.numpy()
    np.savez_compressed(os.path.join(OUT, "compute_loss.npz"), **d)
    print("cls_loss %.6f box_loss %.6f" % (float(cls_loss), float(box_loss)))


if __name__ == "__main__":
    main()
