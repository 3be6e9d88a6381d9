"""Fixture for FPN training: the UNMODIFIED reference Model (odtk/model.py) in training mode on the CPU in fp32, its
BatchNorms converted to FixedBatchNorm2d as odtk/train.py:29 does, on the inputs of gen_golden_head_grads.inputs() (the
deterministic synthetic state_dict of retinanet_examples_b200.model.make_state_dict with livelier head weights, the
seeded image batch and targets).  `model([x, targets])` -> (cls_loss, box_loss), then autograd of cls_loss + box_loss
w.r.t. every parameter.  Stored for the 8 FPN convolutions (fpn.py:26-33): every bias gradient, the per-output-channel
gradient norms of every weight and the full weight gradients of a seeded subset of output channels (the whole weight
gradients would make the file about 5 MB: pyramid6 alone is 256 x 512 x 9), plus the losses.
    python oracle/gen_golden_fpn_grads.py  ->  tests/golden/fpn_grads.npz          TEST INFRASTRUCTURE ONLY."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_import  # noqa: E402
from oracle.gen_golden_head_grads import BACKBONE, CLASSES, inputs  # noqa: E402,F401  (the GPU test imports them here)

OUT = os.path.join(ROOT, "tests", "golden")
LAYERS = ("lateral3", "lateral4", "lateral5", "pyramid6", "pyramid7", "smooth3", "smooth4", "smooth5")
CHANNELS = 4          # output channels stored in full per layer


def layer_channels(name):
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
    for layer in LAYERS:
        name = "backbones.%s.%s" % (BACKBONE, layer)
        gw, gb = params[name + ".weight"].grad, params[name + ".bias"].grad
        ch = layer_channels(name)
        d[name + ".bias"] = gb.numpy()
        d[name + ".channels"] = ch.numpy()
        d[name + ".weight"] = gw[ch].numpy()
        d[name + ".norms"] = gw.flatten(1).norm(dim=1).numpy()
    np.savez_compressed(os.path.join(OUT, "fpn_grads.npz"), **d)
    print("cls_loss %.6f box_loss %.6f" % (float(cls_loss), float(box_loss)))


if __name__ == "__main__":
    main()
