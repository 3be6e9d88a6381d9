"""Golden outputs of the reference's own CUDA kernels (TEST INFRASTRUCTURE ONLY; needs a GPU).

Runs csrc/cuda/{decode,decode_rotate,nms,nms_iou}.cu of the unmodified reference -- compiled by oracle/Makefile into
oracle/_ref/libodtk_ref.so (--use_fast_math, as its setup.py builds them) -- on the seeded inputs of
tests/test_gpu_postproc.py::test_against_reference_cuda_kernels and tests/test_gpu_targets.py::test_iou_matches_reference_cuda_kernel,
and stores what they return in tests/golden/ref_cuda.npz:

    python oracle/gen_golden_refcuda.py [out.npz]
"""
import ctypes
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle  # noqa: E402

DEV = "cuda:0"


def level_case(rng, b, c, h, w, a, mu, nbox=4):
    cls = (1 / (1 + np.exp(-rng.normal(mu, 1.6, size=(b, a * c, h, w))))).astype(np.float32)
    deltas = rng.normal(0, 0.2, size=(b, a * nbox, h, w)).astype(np.float32)
    return cls, deltas


def decode_case(rotated):
    """Inputs of test_against_reference_cuda_kernels: (cls, deltas, anchors, stride)."""
    rng = np.random.default_rng(31)
    A, nbox, stride = (27 if rotated else 9), (6 if rotated else 4), 16
    anchors = (oracle.generate_anchors_rotated_axis(stride, oracle.DEFAULT_RATIOS, oracle.DEFAULT_SCALES, oracle.DEFAULT_ANGLES)
               if rotated else oracle.generate_anchors(stride, oracle.DEFAULT_RATIOS, oracle.DEFAULT_SCALES)).reshape(-1).tolist()
    cls, deltas = level_case(rng, 2, 10, 25, 40, A, -3.5, nbox)
    if rotated:
        th = rng.uniform(-np.pi / 4, np.pi / 4, size=(2, A, 25, 40))
        d = deltas.reshape(2, A, 6, 25, 40); d[:, :, 4] = np.sin(th); d[:, :, 5] = np.cos(th)
    return cls, deltas, anchors, stride


def iou_case():
    """Inputs of test_iou_matches_reference_cuda_kernel: (boxes [5, 8], anchors [295, 8])."""
    rng = np.random.default_rng(8)
    c = rng.uniform(0, 200, (300, 1, 2))
    quads = (c + np.array([[-20, -10], [20, -10], [20, 10], [-20, 10]]) * rng.uniform(0.5, 2, (300, 1, 1))).reshape(300, 8).astype(np.float32)
    return quads[:5].copy(), quads[5:].copy()


def _call(fn, args):
    size = fn(*args, None, ctypes.c_longlong(0), None)
    ws = torch.zeros(size, dtype=torch.uint8, device=DEV)
    torch.cuda.synchronize()
    assert fn(*args, ctypes.c_void_p(ws.data_ptr()), ctypes.c_longlong(size), None) == 0
    torch.cuda.synchronize()


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "ref_cuda.npz")
    L = ctypes.CDLL(os.path.join(ROOT, "oracle", "_ref", "libodtk_ref.so"))
    L.ref_decode.restype = L.ref_nms.restype = L.ref_iou.restype = ctypes.c_longlong
    g = {}
    for rotated in (False, True):
        cls, deltas, anchors, stride = decode_case(rotated)
        tc, td = torch.from_numpy(cls).to(DEV), torch.from_numpy(deltas).to(DEV)
        b, ac, h, w = cls.shape
        nbox, a, top_n = (6 if rotated else 4), len(anchors) // 4, 1000
        s = torch.zeros(b, top_n, device=DEV); bx = torch.zeros(b, top_n, nbox, device=DEV); c = torch.zeros(b, top_n, device=DEV)
        anc = (ctypes.c_float * len(anchors))(*anchors)
        _call(L.ref_decode, [b, ctypes.c_void_p(tc.data_ptr()), ctypes.c_void_p(td.data_ptr()), ctypes.c_void_p(s.data_ptr()),
                             ctypes.c_void_p(bx.data_ptr()), ctypes.c_void_p(c.data_ptr()), h, w, stride, a, ac // a, anc,
                             len(anchors), ctypes.c_float(0.05), top_n, int(rotated)])
        det = 100
        os_ = torch.zeros(b, det, device=DEV); ob = torch.zeros(b, det, nbox, device=DEV); oc = torch.zeros(b, det, device=DEV)
        _call(L.ref_nms, [b, ctypes.c_void_p(s.data_ptr()), ctypes.c_void_p(bx.data_ptr()), ctypes.c_void_p(c.data_ptr()),
                          ctypes.c_void_p(os_.data_ptr()), ctypes.c_void_p(ob.data_ptr()), ctypes.c_void_p(oc.data_ptr()), top_n, det,
                          ctypes.c_float(0.5), int(rotated)])
        r = "rot" if rotated else "axis"
        for k, t in (("dec_scores", s), ("dec_boxes", bx), ("dec_classes", c), ("nms_scores", os_), ("nms_boxes", ob), ("nms_classes", oc)):
            g["%s_%s" % (k, r)] = t.cpu().numpy()
    boxes, anchors = iou_case()
    bt, at = torch.from_numpy(boxes).to(DEV), torch.from_numpy(anchors).to(DEV)
    iou = torch.zeros((anchors.shape[0], boxes.shape[0]), device=DEV)
    torch.cuda.synchronize()
    assert L.ref_iou(ctypes.c_void_p(bt.data_ptr()), ctypes.c_void_p(at.data_ptr()), ctypes.c_void_p(iou.data_ptr()), 5, 295, None) == 0
    torch.cuda.synchronize()
    g["iou"] = iou.cpu().numpy()
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    np.savez_compressed(out, **g)
    print("wrote", out, {k: v.shape for k, v in g.items()})


if __name__ == "__main__":
    main()
