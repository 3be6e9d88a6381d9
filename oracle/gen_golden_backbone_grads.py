"""Fixture for training ResNet stages 3-4: the UNMODIFIED reference Model (odtk/model.py) in training mode on the CPU in
fp32, its BatchNorms converted to FixedBatchNorm2d as odtk/train.py:29 does, on the inputs of
gen_golden_head_grads.inputs() (as gen_golden_fpn_grads.py).  `model([x, targets])` -> (cls_loss, box_loss), then autograd
of cls_loss + box_loss w.r.t. every parameter.  Stored: the losses, the reference's named_parameters() names in order, and
for every layer3 / layer4 convolution weight the per-output-channel gradient norms and the full gradients of four seeded
output channels (the whole gradients would make the file about 40 MB).
    python oracle/gen_golden_backbone_grads.py  ->  tests/golden/backbone_grads.npz          TEST INFRASTRUCTURE ONLY."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_import  # noqa: E402
from oracle.gen_golden_head_grads import BACKBONE, CLASSES, inputs  # noqa: E402,F401  (the GPU test imports them here)

OUT = os.path.join(ROOT, "tests", "golden")
CHANNELS = 4          # output channels stored in full per weight


def stage_weight(name):
    return ".features.layer3." in name or ".features.layer4." in name


def weight_channels(name, cout):
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    return torch.randperm(cout, generator=g)[:CHANNELS].sort().values


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
    d = {"x_sum": np.float64(x.double().sum()), "cls_loss": cls_loss.detach().numpy(),
         "box_loss": box_loss.detach().numpy(), "names": np.array(list(params))}
    for name, p in params.items():
        if not stage_weight(name):
            continue
        gw = p.grad
        ch = weight_channels(name, gw.shape[0])
        d[name + ".channels"] = ch.numpy()
        d[name] = gw[ch].numpy()
        d[name + ".norms"] = gw.flatten(1).norm(dim=1).numpy()
    np.savez_compressed(os.path.join(OUT, "backbone_grads.npz"), **d)
    print("cls_loss %.6f box_loss %.6f" % (float(cls_loss), float(box_loss)))


if __name__ == "__main__":
    main()
