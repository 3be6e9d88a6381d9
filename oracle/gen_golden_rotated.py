"""Fixtures for the rotated training-side target assignment, made in the build container:
    python oracle/gen_golden_rotated.py  ->  tests/golden/snap_rotated.npz
TEST INFRASTRUCTURE ONLY.

The reference's odtk.box.snap_to_anchors_rotated (odtk/box.py:192-252) and odtk.utils.rotate_boxes are imported
UNMODIFIED from /root/reference and run on CPU.  Their only compiled dependency is `iou_cuda` (= odtk._C.iou, the
kernel of csrc/cuda/nms_iou.cu:324-387), absent here: it is replaced by oracle.iou (oracle/odtk_oracle.c:oracle_iou, the
C restatement of that kernel, itself checked against the reference kernel compiled into oracle/_ref on the GPU box by
tests/test_gpu_targets.py::test_iou_matches_reference_cuda_kernel), and torch.cuda.is_available is forced to True for
the duration of the call because the reference binds `iou` only under that condition (box.py:215-216).
Also stores raw iou cases (boxes, anchors, iou) so that the oracle itself is pinned by committed numbers."""
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle, ref_import  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def main():
    odtk = ref_import.import_reference()
    import odtk.box as rbox
    import odtk.utils as rutils

    def iou_cpu(boxes, anchors):
        return [torch.from_numpy(oracle.iou(boxes.numpy().reshape(-1, 8), anchors.numpy().reshape(-1, 8)))]

    rbox.iou_cuda = iou_cpu
    real_avail = torch.cuda.is_available
    ratios, scales = [1.0, 2.0, 0.5], [4 * 2 ** (i / 3) for i in range(3)]
    angles = [-math.pi / 6, 0, math.pi / 6]
    rng = np.random.default_rng(11)
    d, k = {}, 0
    cases = [(32, 10, 7, 6, 5), (64, 6, 5, 3, 3), (16, 12, 8, 12, 80), (128, 3, 2, 1, 4)]
    for (stride, w, h, g, ncls) in cases:
        wh = rng.uniform(1.0 * stride, 6.0 * stride, size=(g, 2))
        xy = rng.uniform(0, [w * stride * 0.8, h * stride * 0.8], size=(g, 2))
        th = rng.uniform(-0.6, 0.6, size=(g, 1))
        cls = rng.integers(0, ncls, size=(g, 1)).astype(np.float64)
        boxes = np.concatenate([np.round(xy), np.round(wh), th, cls], 1).astype(np.float32)
        if k == 1:                       # one box that coincides with an anchor footprint, one axis-aligned
            boxes[0, 4] = 0.0
        anchors = rbox.generate_anchors_rotated(stride, ratios, scales, angles)
        torch.cuda.is_available = lambda: True
        try:
            ct, bt, dp = rbox.snap_to_anchors_rotated(torch.from_numpy(boxes), [w * stride, h * stride], stride, anchors,
                                                      ncls, "cpu", [0.4, 0.5])
            ba, br = rutils.rotate_boxes(torch.from_numpy(boxes[:, :5]))
        finally:
            torch.cuda.is_available = real_avail
        d.update({"c%d_boxes" % k: boxes, "c%d_size" % k: np.array([w * stride, h * stride]), "c%d_stride" % k: stride,
                  "c%d_classes" % k: ncls, "c%d_anchors_axis" % k: anchors[0].numpy(), "c%d_anchors_rot" % k: anchors[1].numpy(),
                  "c%d_cls_target" % k: ct.numpy().astype(np.uint8), "c%d_box_target" % k: bt.numpy(), "c%d_depth" % k: dp.numpy(),
                  "c%d_boxes_axis" % k: ba.numpy(), "c%d_boxes_rot" % k: br.numpy()})
        k += 1
    d["ncases"] = k
    # raw iou known answers (oracle_iou): random quads around shared centres, identical quads, disjoint quads
    q = rng.uniform(0, 100, size=(40, 1, 2)) + rng.uniform(-30, 30, size=(40, 4, 2))
    boxes_q, anchors_q = q[:7].reshape(-1, 8).astype(np.float32), q[7:].reshape(-1, 8).astype(np.float32)
    ax, rot = rbox.generate_anchors_rotated(32, ratios, scales, angles)
    anchors_q = np.concatenate([anchors_q, rot.numpy()[:9] + 40.0, boxes_q[:2]], 0).astype(np.float32)
    d["iou_boxes"], d["iou_anchors"] = boxes_q, anchors_q
    d["iou"] = oracle.iou(boxes_q, anchors_q)
    np.savez_compressed(os.path.join(OUT, "snap_rotated.npz"), **d)
    print("wrote snap_rotated.npz:", k, "cases; foreground anchors per case:",
          [int((d["c%d_depth" % i] > 0).sum()) for i in range(k)], "iou range", float(d["iou"].min()), float(d["iou"].max()))


if __name__ == "__main__":
    main()
