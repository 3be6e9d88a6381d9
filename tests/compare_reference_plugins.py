"""Comparator for BASELINE.json configs[1] / [4] (not collected by pytest; run on an H100):
decode + NMS on the RetinaNet head shapes, OUR sm_90a kernels vs the reference's own csrc/cuda
kernels compiled unmodified for sm_90a (oracle/_ref/libodtk_ref.so), identical fp32 NCHW inputs,
CUDA-event timing, results compared.  Writes one JSON line.

    python tests/compare_reference_plugins.py [--batch 8] [--rotated]
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from retinanet_examples_b200 import _C, box, synth

DEV = "cuda:0"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--rotated", action="store_true")
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    L = ctypes.CDLL(os.path.join(ROOT, "oracle", "_ref", "libodtk_ref.so"))
    L.ref_decode.restype = ctypes.c_longlong
    L.ref_nms.restype = ctypes.c_longlong
    rot, nbox, A = a.rotated, (6 if a.rotated else 4), (27 if a.rotated else 9)
    cls, deltas = synth.head_outputs(a.batch, seed=0, rotated=rot, anchors=A, device=DEV)
    anchors = [(box.generate_anchors_rotated(s, box.DEFAULT_RATIOS, box.DEFAULT_SCALES, box.DEFAULT_ANGLES)[0] if rot
                else box.generate_anchors(s, box.DEFAULT_RATIOS, box.DEFAULT_SCALES)).reshape(-1).tolist() for s in synth.LEVEL_STRIDES]
    B, top_n, det = a.batch, 1000, 100

    def ours():
        d = _C.decode_levels(cls, deltas, anchors, synth.LEVEL_STRIDES, 0.05, top_n, rot)
        return _C.nms(*d, 0.5, det, rot)

    # reference: per level decode (workspace zeroed like torch::zeros in extensions.cpp:94), cat, nms
    ws_sizes = []
    for lvl in range(5):
        _, ac, h, w = cls[lvl].shape
        anc = (ctypes.c_float * len(anchors[lvl]))(*anchors[lvl])
        ws_sizes.append(L.ref_decode(B, None, None, None, None, None, h, w, synth.LEVEL_STRIDES[lvl], A, ac // A, anc,
                                     len(anchors[lvl]), ctypes.c_float(0.05), top_n, int(rot), None, ctypes.c_longlong(0), None))
    nms_ws = L.ref_nms(B, None, None, None, None, None, None, 5 * top_n, det, ctypes.c_float(0.5), int(rot), None, ctypes.c_longlong(0), None)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def reference():
        outs = []
        for lvl in range(5):
            _, ac, h, w = cls[lvl].shape
            s = torch.zeros(B, top_n, device=DEV); bx = torch.zeros(B, top_n, nbox, device=DEV); c = torch.zeros(B, top_n, device=DEV)
            ws = torch.zeros(ws_sizes[lvl], dtype=torch.uint8, device=DEV)
            anc = (ctypes.c_float * len(anchors[lvl]))(*anchors[lvl])
            rc = L.ref_decode(B, ctypes.c_void_p(cls[lvl].data_ptr()), ctypes.c_void_p(deltas[lvl].data_ptr()),
                              ctypes.c_void_p(s.data_ptr()), ctypes.c_void_p(bx.data_ptr()), ctypes.c_void_p(c.data_ptr()), h, w,
                              synth.LEVEL_STRIDES[lvl], A, ac // A, anc, len(anchors[lvl]), ctypes.c_float(0.05), top_n, int(rot),
                              ctypes.c_void_p(ws.data_ptr()), ctypes.c_longlong(ws_sizes[lvl]), stream)
            assert rc == 0
            outs.append((s, bx, c))
        s, bx, c = [torch.cat(t, 1) for t in zip(*outs)]
        os_ = torch.zeros(B, det, device=DEV); ob = torch.zeros(B, det, nbox, device=DEV); oc = torch.zeros(B, det, device=DEV)
        ws = torch.zeros(nms_ws, dtype=torch.uint8, device=DEV)
        rc = L.ref_nms(B, ctypes.c_void_p(s.data_ptr()), ctypes.c_void_p(bx.data_ptr()), ctypes.c_void_p(c.data_ptr()),
                       ctypes.c_void_p(os_.data_ptr()), ctypes.c_void_p(ob.data_ptr()), ctypes.c_void_p(oc.data_ptr()), 5 * top_n, det,
                       ctypes.c_float(0.5), int(rot), ctypes.c_void_p(ws.data_ptr()), ctypes.c_longlong(nms_ws), stream)
        assert rc == 0
        return os_, ob, oc

    def time_it(fn, iters):
        for _ in range(3):
            out = fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters * 1e3 / B, out

    us_ours, o = time_it(ours, a.iters)
    us_ref, r = time_it(reference, max(3, a.iters // 4))
    o = [t.cpu().numpy() for t in o]
    r = [t.cpu().numpy() for t in r]
    keep = r[0] > 0
    same_scores = float((o[0][keep] == r[0][keep]).mean())
    max_box = float(np.abs(o[1][keep] - r[1][keep]).max()) if same_scores == 1.0 else None
    print(json.dumps({"workload": "decode+NMS, ResNet50FPN head shapes 3x800x1280, batch %d%s" % (B, ", rotated" if rot else ""),
                      "ours_us_per_image": round(us_ours, 2), "reference_cuda_plugins_us_per_image": round(us_ref, 2),
                      "speedup": round(us_ref / us_ours, 1), "kept_scores_identical_fraction": same_scores,
                      "max_abs_box_diff_vs_fast_math_reference": max_box,
                      "reference": "csrc/cuda/{decode,decode_rotate,nms,nms_iou}.cu unmodified, nvcc -gencode arch=compute_90a,code=sm_90a --use_fast_math"}))


if __name__ == "__main__":
    main()
