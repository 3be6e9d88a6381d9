"""Host-side mirror of the reference's odtk/box.py for the inference hot path: anchor tables
(setup-time, CPU) and the decode / nms / nms_rotated dispatchers, which here ALWAYS run the
sm_90a kernels (the reference dispatches to odtk._C when torch.cuda.is_available(),
odtk/box.py:262,315,373, and otherwise to a CPU fallback -- this package has no fallback)."""
import math

import numpy as np
import torch

from . import _C


def generate_anchors(stride, ratio_vals, scales_vals, angles_vals=None):
    """Anchor coordinates [A, 4] (x1, y1, x2, y2) for one pyramid level.
    Reference: odtk/box.py:8-20; known answers: extras/cppapi/export.cpp:69-75."""
    f = np.float32
    nr, ns = len(ratio_vals), len(scales_vals)
    scales = np.repeat(np.asarray(scales_vals, dtype=f), nr)[:, None]       # scale-major, ratio-minor
    ratios = np.tile(np.asarray(ratio_vals, dtype=f), ns)
    side = np.full((nr * ns, 2), stride, dtype=f)
    w = np.sqrt(side[:, 0] * side[:, 1] / ratios).astype(f)
    wh = np.stack([w, (w * ratios).astype(f)], axis=1)
    lo = (f(0.5) * (side - wh * scales)).astype(f)
    hi = (f(0.5) * (side + wh * scales)).astype(f)
    return torch.from_numpy(np.concatenate([lo, hi], axis=1))


def _order_points(quads):
    """Order 4 corners as (top-left, top-right, bottom-right, bottom-left).
    Reference: odtk/utils.py:15-31."""
    out = []
    for pt in quads:
        by_x = pt[torch.argsort(pt[:, 0])]
        left, right = by_x[:2], by_x[2:]
        left = left[torch.argsort(left[:, 1])]
        tl, bl = left[0], left[1]
        dist = torch.cdist(tl[None], right)[0]
        far = right[torch.argsort(dist, descending=True)]
        br, tr = far[0], far[1]
        out.append(torch.stack([tl, tr, br, bl]))
    return torch.stack(out)


def generate_anchors_rotated(stride, ratio_vals, scales_vals, angles_vals):
    """Returns (anchors_axis [A*len(angles), 4], anchors_rotated [A*len(angles), 8]).
    Only anchors_axis is consumed by decode (odtk/box.py:258-259, decode_rotate.cu:139).
    Reference: odtk/box.py:23-64; known answers: extras/cppapi/export.cpp:79-85."""
    f = torch.float32
    nr, ns, na = len(ratio_vals), len(scales_vals), len(angles_vals)
    scales = torch.tensor(scales_vals, dtype=f).repeat_interleave(nr)[:, None]
    ratios = torch.tensor(list(ratio_vals) * ns, dtype=f)
    side = torch.full((nr * ns, 2), float(stride), dtype=f)
    w = torch.round(torch.sqrt(side[:, 0] * side[:, 1] / ratios))
    wh = torch.stack([w, torch.round(w * ratios)], dim=1)
    p0 = 0.5 * (side - wh * scales)
    p2 = 0.5 * (side + wh * scales) - 1
    p1 = p0 + (p2 - p0) * torch.tensor([0.0, 1.0])
    p3 = p0 + (p2 - p0) * torch.tensor([1.0, 0.0])
    angles = torch.tensor(angles_vals, dtype=f)
    rot = torch.stack([torch.stack([torch.cos(angles), torch.sin(angles)], dim=1),
                       torch.stack([-torch.sin(angles), torch.cos(angles)], dim=1)], dim=1)  # [na, 2, 2]
    half = stride / 2 - 0.5

    def spin(pts):
        r = torch.matmul(rot, pts.t() - half) + half            # [na, 2, n]
        return r.permute(0, 2, 1).contiguous().view(-1, 2)

    corners = torch.stack([spin(p0), spin(p1), spin(p2), spin(p3)], dim=1)
    anchors_axis = torch.cat([p0.repeat(na, 1), p2.repeat(na, 1)], dim=1)
    anchors_rotated = _order_points(corners).view(-1, 8)
    return anchors_axis, anchors_rotated


def decode(all_cls_head, all_box_head, stride=1, threshold=0.05, top_n=1000, anchors=None, rotated=False):
    """Box decoding and filtering of one pyramid level for the whole batch.
    Reference: odtk/box.py:255-264 -> odtk._C.decode (the `.float()` casts are kept)."""
    if rotated:
        anchors = anchors[0]
    flat = anchors.reshape(-1).tolist() if anchors is not None else []
    return _C.decode(all_cls_head.float().contiguous(), all_box_head.float().contiguous(), flat, stride,
                     threshold, top_n, rotated)


def nms(all_scores, all_boxes, all_classes, nms=0.5, ndetections=100):
    """Per-image non-maximum suppression.  Reference: odtk/box.py:312-317 -> odtk._C.nms."""
    return _C.nms(all_scores.float().contiguous(), all_boxes.float().contiguous(),
                  all_classes.float().contiguous(), nms, ndetections, False)


def nms_rotated(all_scores, all_boxes, all_classes, nms=0.5, ndetections=100):
    """Rotated-box NMS.  Reference: odtk/box.py:370-375 -> odtk._C.nms(..., rotated=True)."""
    return _C.nms(all_scores.float().contiguous(), all_boxes.float().contiguous(),
                  all_classes.float().contiguous(), nms, ndetections, True)


DEFAULT_RATIOS = [1.0, 2.0, 0.5]
DEFAULT_SCALES = [4 * 2 ** (i / 3) for i in range(3)]
DEFAULT_ANGLES = [-math.pi / 6, 0, math.pi / 6]


def snap_to_anchors_batch(targets, size, stride, anchors, num_classes, anchor_ious, dense=True):
    """Target assignment for a whole batch at one pyramid level in ONE launch (odtk_snap_to_anchors).
    targets [B, G, 5] fp32 CUDA (x, y, w, h, class; class <= -1 = padding row, skipped on the device);
    size = (H, W) of the head tensors; anchors [A, 4].  Returns (cls_target [B,A,C,H,W] or None when
    dense=False, box_target [B,A,4,H,W], depth [B,A,1,H,W], cls_index [B,A,H,W] int32) -- the stacked results of
    Model._extract_targets (odtk/model.py:167-184) plus the class-index targets loss.FocalLoss accepts."""
    import ctypes
    from . import _lib
    if not (targets.is_cuda and targets.dtype == torch.float32 and targets.dim() == 3 and targets.size(2) == 5):
        raise ValueError("targets must be a CUDA fp32 [B, G, 5] tensor: there is no CPU path")
    targets = targets.contiguous()
    batch, g = targets.size(0), targets.size(1)
    h, w = int(size[0]), int(size[1])
    a = anchors.reshape(-1, 4)
    na, dev = a.size(0), targets.device
    host = (ctypes.c_float * (4 * na))(*[float(v) for v in a.reshape(-1).tolist()])
    cls_target = torch.empty((batch, na, num_classes, h, w), dtype=torch.float32, device=dev) if dense else None
    box_target = torch.empty((batch, na, 4, h, w), dtype=torch.float32, device=dev)
    depth = torch.empty((batch, na, 1, h, w), dtype=torch.float32, device=dev)
    cls_index = torch.empty((batch, na, h, w), dtype=torch.int32, device=dev)
    _lib.check(_lib.lib().odtk_snap_to_anchors(
        ctypes.c_void_p(targets.data_ptr()) if g else None, batch, g, h, w, int(stride),
        ctypes.cast(host, ctypes.POINTER(ctypes.c_float)), na, int(num_classes), float(anchor_ious[0]), float(anchor_ious[1]),
        ctypes.c_void_p(cls_target.data_ptr()) if dense else None, ctypes.c_void_p(box_target.data_ptr()),
        ctypes.c_void_p(depth.data_ptr()), ctypes.c_void_p(cls_index.data_ptr()),
        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "snap_to_anchors")
    return cls_target, box_target, depth, cls_index


def snap_to_anchors(boxes, size, stride, anchors, num_classes, device, anchor_ious):
    """'Snap target boxes (x, y, w, h) to anchors' -- odtk/box.py:134-186, same signature and results:
    boxes [G, 5] (x, y, w, h, class) of ONE image, size = [W*stride, H*stride]; returns
    (cls_target [A,C,H,W], box_target [A,4,H,W], depth [A,1,H,W])."""
    width, height = int(size[0] / stride), int(size[1] / stride)
    t = boxes.to(device=device, dtype=torch.float32).reshape(1, -1, 5)
    cls_target, box_target, depth, _ = snap_to_anchors_batch(t, (height, width), stride, anchors, num_classes, anchor_ious)
    return cls_target[0], box_target[0], depth[0]


# ---- rotated-box target assignment (reference odtk/box.py:80-96,189-252, odtk/utils.py:33-80) ----
def rotate_boxes(boxes, points=False):
    """Target boxes (xmin, ymin, width, height, theta) -> (boxes_axis [G, 6] = (x1, y1, x2, y2, sin, cos),
    boxes_rotated [G, 8] = the four rotated corners ordered tl, tr, br, bl).  Reference: odtk/utils.py:33-80."""
    th = boxes[:, 4]
    u = torch.stack([torch.cos(th), torch.sin(th)], dim=1)
    l = torch.stack([-torch.sin(th), torch.cos(th)], dim=1)
    R = torch.stack([u, l], dim=1)                                   # [G, 2, 2]
    if points:
        cents = torch.stack([(boxes[:, 0] + boxes[:, 2]) / 2, (boxes[:, 1] + boxes[:, 3]) / 2], 1)
        x0, y0, x1, y1 = boxes[:, 0], boxes[:, 1], boxes[:, 2], boxes[:, 3]
    else:
        cents = torch.stack([boxes[:, 0] + boxes[:, 2] / 2, boxes[:, 1] + boxes[:, 3] / 2], 1)
        x0, y0, x1, y1 = boxes[:, 0], boxes[:, 1], boxes[:, 0] + boxes[:, 2], boxes[:, 1] + boxes[:, 3]
    corners = torch.stack([torch.stack([x0, y0], 1), torch.stack([x1, y0], 1), torch.stack([x1, y1], 1),
                           torch.stack([x0, y1], 1)], dim=1)         # [G, 4, 2]
    # per box: R @ (corner - centre) + centre (the reference builds the full [G, 2, G] product and takes its diagonal)
    rot = torch.matmul(R[:, None], (corners - cents[:, None])[..., None])[..., 0] + cents[:, None]
    boxes_axis = torch.cat([boxes[:, :2], boxes[:, :2] + boxes[:, 2:4] - 1,
                            torch.sin(boxes[:, -1, None]), torch.cos(boxes[:, -1, None])], 1)
    return boxes_axis, _order_points(rot).view(-1, 8)


def box2delta_rotated(boxes, anchors):
    """'Convert boxes to deltas from anchors' -- odtk/box.py:80-94."""
    anchors_wh = anchors[:, 2:4] - anchors[:, :2] + 1
    anchors_ctr = anchors[:, :2] + 0.5 * anchors_wh
    boxes_wh = boxes[:, 2:4] - boxes[:, :2] + 1
    boxes_ctr = boxes[:, :2] + 0.5 * boxes_wh
    return torch.cat([(boxes_ctr - anchors_ctr) / anchors_wh, torch.log(boxes_wh / anchors_wh),
                      boxes[:, 4, None], boxes[:, 5, None]], 1)


def snap_to_anchors_rotated(boxes, size, stride, anchors, num_classes, device, anchor_ious):
    """'Snap target boxes (x, y, w, h, a) to anchors' -- odtk/box.py:192-252, same signature and results.
    boxes [G, 6] (x, y, w, h, theta, class) of ONE image; anchors = (anchors_axis [A, 4], anchors_rotated [A, 8]) from
    generate_anchors_rotated; size = [W*stride, H*stride].  The A*H*W x G polygon IoUs run on the sm_90a kernel
    (_C.iou -> odtk_iou); the arg-max / delta / scatter bookkeeping are the reference's own tensor expressions on the
    device.  Returns (cls_target [A, C, H, W], box_target [A, 6, H, W], depth [A, 1, H, W])."""
    anchors_axis, anchors_rotated = anchors
    num_anchors = anchors_rotated.size()[0] if anchors_rotated is not None else 1
    width, height = int(size[0] / stride), int(size[1] / stride)
    if boxes.nelement() == 0:
        return (torch.zeros([num_anchors, num_classes, height, width], device=device),
                torch.zeros([num_anchors, 6, height, width], device=device),
                torch.zeros([num_anchors, 1, height, width], device=device))
    boxes = boxes.to(device=device, dtype=torch.float32)
    boxes, classes = boxes.split(5, dim=1)
    boxes_axis, boxes_rotated = rotate_boxes(boxes)
    anchors_axis = anchors_axis.to(device=device, dtype=torch.float32)
    anchors_rotated = anchors_rotated.to(device=device, dtype=torch.float32)
    xs = torch.arange(0, size[0], stride, device=device, dtype=classes.dtype)
    ys = torch.arange(0, size[1], stride, device=device, dtype=classes.dtype)
    x, y = torch.meshgrid(xs, ys, indexing="ij")
    xy_2corners = torch.stack((x, y, x, y), 2).unsqueeze(0)
    xy_4corners = torch.stack((x, y, x, y, x, y, x, y), 2).unsqueeze(0)
    anchors_axis = (xy_2corners.to(torch.float) + anchors_axis.view(-1, 1, 1, 4)).contiguous().view(-1, 4)
    anchors_rotated = (xy_4corners.to(torch.float) + anchors_rotated.view(-1, 1, 1, 8)).contiguous().view(-1, 8)
    overlap = _C.iou(boxes_rotated.contiguous().view(-1), anchors_rotated.contiguous().view(-1))[0]
    overlap, indices = overlap.max(1)                                 # best box per anchor
    box_target = box2delta_rotated(boxes_axis[indices], anchors_axis)
    box_target = box_target.view(num_anchors, 1, width, height, 6).transpose(1, 4).transpose(2, 3)
    box_target = box_target.squeeze().contiguous()
    depth = torch.ones_like(overlap, device=device) * -1
    depth[overlap < anchor_ious[0]] = 0                               # background
    depth[overlap >= anchor_ious[1]] = classes[indices][overlap >= anchor_ious[1]].squeeze() + 1   # objects
    depth = depth.view(num_anchors, width, height).transpose(1, 2).contiguous()
    cls_target = torch.zeros((anchors_axis.size()[0], num_classes + 1), device=device, dtype=boxes_axis.dtype)
    classes = classes[indices].long().view(-1, 1)
    classes[overlap < anchor_ious[0]] = num_classes                   # background has no class
    cls_target.scatter_(1, classes, 1)
    cls_target = cls_target[:, :num_classes].view(-1, 1, width, height, num_classes)
    cls_target = cls_target.transpose(1, 4).transpose(2, 3).squeeze().contiguous()
    return (cls_target.view(num_anchors, num_classes, height, width), box_target.view(num_anchors, 6, height, width),
            depth.view(num_anchors, 1, height, width))
