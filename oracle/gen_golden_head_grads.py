"""Fixture for head training: the UNMODIFIED reference Model (odtk/model.py) in training mode on the CPU in fp32, its
BatchNorms converted to FixedBatchNorm2d as odtk/train.py:29 does, loaded with the deterministic synthetic state_dict of
retinanet_examples_b200.model.make_state_dict.  `model([x, targets])` -> (cls_loss, box_loss), then autograd of
cls_loss + box_loss w.r.t. the head parameters.  Stored: the losses, the full gradients of the two final layers, every
bias gradient, and for the eight tower layers the per-output-channel gradient norms plus the full gradients of a seeded
subset of output channels (the whole tower gradients would make the file 8 MB).
    python oracle/gen_golden_head_grads.py  ->  tests/golden/head_grads.npz          TEST INFRASTRUCTURE ONLY."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_import  # noqa: E402
from retinanet_examples_b200.model import make_state_dict  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
BACKBONE, CLASSES, SEED, SHAPE = "ResNet18FPN", 2, 31, (2, 3, 256, 384)
CHANNELS = 4          # tower output channels stored in full per layer


def inputs():
    """The seeded image batch, targets ([x, y, w, h, class], -1 rows padding) and head-weight state dict of the fixture;
    the GPU test rebuilds them from the same seeds."""
    g = torch.Generator().manual_seed(SEED)
    sd = make_state_dict(BACKBONE, CLASSES, 9, False, SEED)
    for k in sd:       # livelier heads than the init's 0.01 std, so every tower layer's gradient is far from zero
        if k.startswith(("cls_head", "box_head")) and k.endswith("weight"):
            sd[k] = torch.randn(sd[k].shape, generator=g) * 0.03
    x = torch.randn(SHAPE, generator=g)
    t = torch.tensor([[[20., 30., 160., 90., 1.], [200., 40., 120., 150., 0.], [40., 150., 60., 60., 1.]],
                      [[10., 10., 300., 200., 0.], [250., 160., 80., 70., 1.], [-1., -1., -1., -1., -1.]]])
    return sd, x, t


def tower_channels(name):
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    return torch.randperm(256, generator=g)[:CHANNELS].sort().values


def main():
    odtk = ref_import.import_reference()
    from odtk.backbones.layers import convert_fixedbn_model
    sd, x, t = inputs()
    m = odtk.model.Model(BACKBONE, classes=CLASSES)
    full = m.state_dict()
    full.update(sd)
    m.load_state_dict(full)
    m = convert_fixedbn_model(m)
    m.train()
    cls_loss, box_loss = m([x, t])
    (cls_loss + box_loss).backward()
    params = dict(m.named_parameters())
    d = {"x_sum": np.float64(x.double().sum()), "targets": t.numpy(),
         "cls_loss": cls_loss.detach().numpy(), "box_loss": box_loss.detach().numpy()}
    for head in ("cls_head", "box_head"):
        for i in (0, 2, 4, 6, 8):
            name = "%s.%d" % (head, i)
            gw, gb = params[name + ".weight"].grad, params[name + ".bias"].grad
            d[name + ".bias"] = gb.numpy()
            if i == 8:
                d[name + ".weight"] = gw.numpy()
            else:
                ch = tower_channels(name)
                d[name + ".channels"] = ch.numpy()
                d[name + ".weight"] = gw[ch].numpy()
                d[name + ".norms"] = gw.flatten(1).norm(dim=1).numpy()
    np.savez_compressed(os.path.join(OUT, "head_grads.npz"), **d)
    print("cls_loss %.6f box_loss %.6f" % (float(cls_loss), float(box_loss)))


if __name__ == "__main__":
    main()
