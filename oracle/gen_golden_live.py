"""Golden outputs of the unmodified reference on the CPU (TEST INFRASTRUCTURE ONLY; needs the reference sources,
see oracle/ref_import.py): the ResNet18FPN head outputs of test_model_oracle.py::test_model_ref_against_live_reference and
the box.nms trials of test_oracle_golden.py::test_oracle_against_live_reference_nms, stored in tests/golden/live_ref.npz.

    python oracle/gen_golden_live.py [out.npz]
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import gen_golden_model, ref_import  # noqa: E402


def nms_trials():
    """Seeded inputs of the nms comparison: three (scores [1, 300], boxes [1, 300, 4], classes [1, 300])."""
    rng = np.random.default_rng(7)
    out = []
    for _ in range(3):
        n = 300
        ctr = rng.uniform(0, 300, (1, n, 2))
        wh = rng.uniform(20, 100, (1, n, 2))
        b = np.concatenate([ctr - wh / 2, ctr + wh / 2], -1).astype(np.float32)
        s = rng.uniform(0.01, 1, (1, n)).astype(np.float32)
        c = rng.integers(0, 3, (1, n)).astype(np.float32)
        out.append((s, b, c))
    return out


def model_input():
    return torch.randn((1, 3, 128, 128), generator=torch.Generator().manual_seed(5))


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "live_ref.npz")
    odtk = ref_import.import_reference()
    g = {}
    cls, box, _ = gen_golden_model.reference_heads(odtk, "ResNet18FPN", 4, 77, model_input())
    for i, (c, b) in enumerate(zip(cls, box)):
        g["cls%d" % i], g["box%d" % i] = c.numpy(), b.numpy()
    for t, (s, b, c) in enumerate(nms_trials()):
        rs, rb, rc = [x.numpy() for x in odtk.box.nms(torch.from_numpy(s), torch.from_numpy(b), torch.from_numpy(c), 0.5, 100)]
        g["nms%d_scores" % t], g["nms%d_boxes" % t], g["nms%d_classes" % t] = rs, rb, rc
    np.savez_compressed(out, **g)
    print("wrote", out, {k: v.shape for k, v in g.items()})


if __name__ == "__main__":
    main()
