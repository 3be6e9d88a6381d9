"""Mirror of the reference's compiled extension module `odtk._C` (csrc/extensions.cpp:184-201):
`decode`, `nms` with the same signatures, argument meaning, shapes, dtypes and error behaviour
(RuntimeError on non-CUDA / non-contiguous input, extensions.cpp:42-44), implemented by the
sm_90a kernels behind the C ABI; `iou` (extensions.cpp:47-67) likewise.  `Engine` (TensorRT) is outside the hot path."""
import ctypes

import torch

from . import _lib


def _check_input(x, name):
    if not isinstance(x, torch.Tensor) or not x.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor" % name)
    if not x.is_contiguous():
        raise RuntimeError("%s must be contiguous" % name)
    if x.dtype != torch.float32:
        raise RuntimeError("%s must be float32" % name)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _workspace(nbytes, device):
    return torch.empty(int(nbytes), dtype=torch.uint8, device=device)


def decode(cls_head, box_head, anchors, scale, score_thresh, top_n, rotated=False,
           out=None, out_offset=0):
    """odtk._C.decode (csrc/extensions.cpp:69-115).
    cls_head [B, A*C, H, W], box_head [B, A*4|6, H, W] fp32 CUDA contiguous; anchors: flat list of
    4*A floats; returns [scores [B, top_n], boxes [B, top_n, 4|6], classes [B, top_n]].
    `out`/`out_offset` (extension): write into rows of pre-allocated [B, S], [B, S, nbox], [B, S]
    buffers at column out_offset (replaces the torch.cat of odtk/model.py:164)."""
    _check_input(cls_head, "cls_head")
    _check_input(box_head, "box_head")
    L = _lib.lib()
    nbox = 6 if rotated else 4
    anchors = [float(a) for a in anchors]
    batch = cls_head.size(0)
    num_anchors = len(anchors) // 4 if anchors else box_head.size(1) // nbox
    num_classes = cls_head.size(1) // num_anchors
    height, width = cls_head.size(2), cls_head.size(3)
    if out is None:
        scores = torch.zeros((batch, top_n), dtype=torch.float32, device=cls_head.device)
        boxes = torch.zeros((batch, top_n, nbox), dtype=torch.float32, device=cls_head.device)
        classes = torch.zeros((batch, top_n), dtype=torch.float32, device=cls_head.device)
        stride = top_n
    else:
        scores, boxes, classes = out
        stride = scores.size(1)
    inputs = _lib.ptr_array([cls_head.data_ptr(), box_head.data_ptr()])
    outputs = _lib.ptr_array([scores.data_ptr(), boxes.data_ptr(), classes.data_ptr()])
    anc = (ctypes.c_float * max(1, len(anchors)))(*anchors)
    args = (batch, inputs, outputs, height, width, int(scale), num_anchors, num_classes, anc, len(anchors),
            float(score_thresh), int(top_n), nbox, stride, int(out_offset))
    size = _lib.check(L.odtk_decode_ex(*args, None, 0, None), "decode (workspace query)")
    scratch = _workspace(size, cls_head.device)
    _lib.check(L.odtk_decode_ex(*args, ctypes.c_void_p(scratch.data_ptr()), size, _stream()), "decode")
    return [scores, boxes, classes]


def decode_levels(cls_heads, box_heads, anchors, scales, score_thresh, top_n, rotated=False):
    """All pyramid levels of the batch in three launches (H100-native addition, see
    odtk_decode_levels in include/odtk_b200.h).  cls_heads / box_heads: lists of per-level
    tensors as for `decode`; anchors: list of flat per-level lists; scales: per-level strides.
    Returns [scores [B, L*top_n], boxes [B, L*top_n, 4|6], classes [B, L*top_n]] == the torch.cat
    over levels of the per-level `decode` results (odtk/model.py:164)."""
    L = _lib.lib()
    nl = len(cls_heads)
    nbox = 6 if rotated else 4
    for c, b in zip(cls_heads, box_heads):
        _check_input(c, "cls_head")
        _check_input(b, "box_head")
    batch, dev = cls_heads[0].size(0), cls_heads[0].device
    na_floats = len(anchors[0]) if anchors and anchors[0] is not None else 0
    num_anchors = na_floats // 4 if na_floats else box_heads[0].size(1) // nbox
    num_classes = cls_heads[0].size(1) // num_anchors
    levels = (_lib.Level * nl)()
    keep = []
    for i in range(nl):
        anc = (ctypes.c_float * max(1, na_floats))(*[float(a) for a in (anchors[i] if na_floats else [])])
        keep.append(anc)
        levels[i].scores, levels[i].deltas = cls_heads[i].data_ptr(), box_heads[i].data_ptr()
        levels[i].height, levels[i].width, levels[i].scale = cls_heads[i].size(2), cls_heads[i].size(3), int(scales[i])
        levels[i].anchors = ctypes.cast(anc, ctypes.POINTER(ctypes.c_float))
    scores = torch.empty((batch, nl * top_n), dtype=torch.float32, device=dev)
    boxes = torch.empty((batch, nl * top_n, nbox), dtype=torch.float32, device=dev)
    classes = torch.empty((batch, nl * top_n), dtype=torch.float32, device=dev)
    outputs = _lib.ptr_array([scores.data_ptr(), boxes.data_ptr(), classes.data_ptr()])
    args = (batch, nl, ctypes.cast(levels, ctypes.c_void_p), num_anchors, num_classes, na_floats, float(score_thresh),
            int(top_n), nbox, outputs, nl * top_n, 0)
    size = _lib.check(L.odtk_decode_levels(*args, None, 0, None), "decode_levels (workspace query)")
    scratch = _workspace(size, dev)
    _lib.check(L.odtk_decode_levels(*args, ctypes.c_void_p(scratch.data_ptr()), size, _stream()), "decode_levels")
    return [scores, boxes, classes]


class FusedDecode:
    """The two halves of odtk_decode_fused_begin / _finish (include/odtk_b200.h) for one fixed batch and
    pyramid geometry.  `begin()` zeroes the counters and returns one CandSink per level, to be handed to the
    class head's last convolution (engine.conv2d(..., out_mode=OUT_CANDIDATES, sink=...)); `finish(box_heads)`
    returns what decode_levels would have returned for the dense score maps.  The workspace is owned by the
    object, so its addresses are stable across CUDA-graph replays."""

    def __init__(self, batch, sizes, num_anchors, num_classes, anchors, scales, score_thresh, top_n, rotated, device):
        self.batch, self.nl, self.nbox = int(batch), len(sizes), 6 if rotated else 4
        self.num_anchors, self.num_classes = int(num_anchors), int(num_classes)
        self.thresh, self.top_n, self.device = float(score_thresh), int(top_n), device
        self.na_floats = len(anchors[0]) if anchors and anchors[0] is not None else 0
        self.levels = (_lib.Level * self.nl)()
        self._keep = []
        for i, (h, w) in enumerate(sizes):
            anc = (ctypes.c_float * max(1, self.na_floats))(*[float(a) for a in (anchors[i] if self.na_floats else [])])
            self._keep.append(anc)
            self.levels[i].scores, self.levels[i].deltas = None, None
            self.levels[i].height, self.levels[i].width, self.levels[i].scale = int(h), int(w), int(scales[i])
            self.levels[i].anchors = ctypes.cast(anc, ctypes.POINTER(ctypes.c_float))
        self.sinks = (_lib.CandSink * self.nl)()
        L = _lib.lib()
        self.size = _lib.check(L.odtk_decode_fused_begin(*self._begin_args(), None, 0, None), "decode_fused (workspace query)")
        self.scratch = _workspace(self.size, device)

    def _begin_args(self):
        return (self.batch, self.nl, ctypes.cast(self.levels, ctypes.c_void_p), self.num_anchors, self.num_classes,
                self.thresh, self.top_n, ctypes.cast(self.sinks, ctypes.c_void_p))

    def begin(self):
        _lib.check(_lib.lib().odtk_decode_fused_begin(*self._begin_args(), ctypes.c_void_p(self.scratch.data_ptr()),
                                                      self.size, _stream()), "decode_fused_begin")
        return self.sinks

    def finish(self, box_heads):
        for i, b in enumerate(box_heads):
            _check_input(b, "box_head")
            self.levels[i].deltas = b.data_ptr()
        n = self.nl * self.top_n
        scores = torch.empty((self.batch, n), dtype=torch.float32, device=self.device)
        boxes = torch.empty((self.batch, n, self.nbox), dtype=torch.float32, device=self.device)
        classes = torch.empty((self.batch, n), dtype=torch.float32, device=self.device)
        outputs = _lib.ptr_array([scores.data_ptr(), boxes.data_ptr(), classes.data_ptr()])
        _lib.check(_lib.lib().odtk_decode_fused_finish(
            self.batch, self.nl, ctypes.cast(self.levels, ctypes.c_void_p), self.num_anchors, self.num_classes,
            self.na_floats, self.thresh, self.top_n, self.nbox, outputs, n, 0,
            ctypes.c_void_p(self.scratch.data_ptr()), self.size, _stream()), "decode_fused_finish")
        return [scores, boxes, classes]


def nms(scores, boxes, classes, nms_thresh, detections_per_im, rotated=False, return_index=False,
        fixed_angle=False, packed=None, gather=None):
    """odtk._C.nms (csrc/extensions.cpp:117-158).
    scores [B, N], boxes [B, N, 4|6], classes [B, N] fp32 CUDA contiguous; returns
    [scores [B, D], boxes [B, D, 4|6], classes [B, D]] (+ int32 kept positions [B, D] when
    return_index, an extension used by the parity tests).  The kernel writes every output slot, so the outputs are
    allocated uninitialised (the reference zero-fills them first, extensions.cpp:128-130).
    Extensions: `packed` [B, D, 2 + nbox] fp32 receives the (score, box..., class) rows; `gather` (a peer.PeerGather)
    makes the kernel push those rows into every rank's gather buffer and completes the exchange (odtk_nms_gather)."""
    _check_input(scores, "scores")
    _check_input(boxes, "boxes")
    _check_input(classes, "classes")
    L = _lib.lib()
    nbox = 6 if rotated else 4
    batch, count = scores.size(0), scores.size(1)
    dev = scores.device
    out_scores = torch.empty((batch, detections_per_im), dtype=torch.float32, device=dev)
    out_boxes = torch.empty((batch, detections_per_im, nbox), dtype=torch.float32, device=dev)
    out_classes = torch.empty((batch, detections_per_im), dtype=torch.float32, device=dev)
    out_index = torch.empty((batch, detections_per_im), dtype=torch.int32, device=dev) if return_index else None
    inputs = _lib.ptr_array([scores.data_ptr(), boxes.data_ptr(), classes.data_ptr()])
    outputs = _lib.ptr_array([out_scores.data_ptr(), out_boxes.data_ptr(), out_classes.data_ptr()])
    idx_ptr = ctypes.c_void_p(out_index.data_ptr()) if return_index else None
    if packed is not None:
        _check_input(packed, "packed")
        if tuple(packed.shape) != (batch, detections_per_im, 2 + nbox):
            raise RuntimeError("packed must be [B, D, 2 + nbox]")
    if gather is not None and (gather.batch != batch or gather.det != detections_per_im or gather.nbox != nbox):
        raise RuntimeError("gather buffers were sized for another batch / detections / box format")
    args = (batch, inputs, outputs, count, int(detections_per_im), float(nms_thresh), nbox, int(bool(fixed_angle)),
            idx_ptr, ctypes.c_void_p(packed.data_ptr()) if packed is not None else None,
            ctypes.byref(gather.desc) if gather is not None else None)
    size = _lib.check(L.odtk_nms_gather(*args, None, 0, None), "nms (workspace query)")
    scratch = _workspace(size, dev)
    _lib.check(L.odtk_nms_gather(*args, ctypes.c_void_p(scratch.data_ptr()), size, _stream()), "nms")
    if gather is not None:
        _lib.check(L.odtk_gather_wait(ctypes.byref(gather.desc), batch, _stream()), "gather_wait")
        if not torch.cuda.is_current_stream_capturing():      # a captured launch runs at replay time (Model counts those)
            gather.steps += 1
    res = [out_scores, out_boxes, out_classes]
    if return_index:
        res.append(out_index)
    return res


def iou(boxes, anchors):
    """odtk._C.iou (csrc/extensions.cpp:47-67): polygon IoU of rotated boxes against rotated anchors.
    boxes: flat (or [..., 8]) fp32 CUDA tensor of num_boxes quadrilaterals (4 corners x (x, y)); anchors likewise.
    Returns [Tensor[num_anchors, num_boxes]] -- a one-element list, as the reference does."""
    _check_input(boxes, "boxes")
    _check_input(anchors, "anchors")
    num_boxes, num_anchors = boxes.numel() // 8, anchors.numel() // 8
    out = torch.empty((num_anchors, num_boxes), dtype=torch.float32, device=boxes.device)
    inputs = _lib.ptr_array([boxes.data_ptr(), anchors.data_ptr()])
    outputs = _lib.ptr_array([out.data_ptr()])
    _lib.check(_lib.lib().odtk_iou(inputs, outputs, num_boxes, num_anchors, _stream()), "iou")
    return [out]
