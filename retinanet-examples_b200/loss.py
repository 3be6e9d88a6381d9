"""Host-side mirror of the reference's odtk/loss.py FocalLoss on the fused sm_90a kernel
(odtk_focal_loss in include/odtk_b200.h).  `FocalLoss()(pred_logits, target)` returns the
element-wise loss like the reference module; `focal_loss_sum` is the fused training form
(masked sum + gradient in one pass, usable with autograd)."""
import ctypes

import torch

from . import _lib


def _launch(logits, target, mask, cls_index, num_classes, hw, alpha, gamma, grad_scale, want_elem, want_grad):
    if not logits.is_cuda:
        raise RuntimeError("pred_logits must be a CUDA tensor")
    L = _lib.lib()
    x = logits.float().contiguous()
    n = x.numel()
    elem = torch.empty_like(x) if want_elem else None
    grad = torch.empty_like(x) if want_grad else None
    total = torch.empty(1, dtype=torch.float32, device=x.device)

    def p(t):
        return ctypes.c_void_p(t.data_ptr()) if t is not None else None
    args = (p(x), p(target), p(mask), p(cls_index), n, int(num_classes), int(hw), float(alpha), float(gamma),
            float(grad_scale), p(elem), p(total), p(grad))
    size = _lib.check(L.odtk_focal_loss(*args, None, 0, None), "focal_loss (workspace query)")
    ws = torch.empty(int(size), dtype=torch.uint8, device=x.device)
    _lib.check(L.odtk_focal_loss(*args, ctypes.c_void_p(ws.data_ptr()), size,
                                 ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "focal_loss")
    return total, elem, grad


class FocalLoss:
    'Focal Loss - https://arxiv.org/abs/1708.02002 (reference: odtk/loss.py:5-18)'

    def __init__(self, alpha=0.25, gamma=2):
        self.alpha, self.gamma = alpha, gamma

    def forward(self, pred_logits, target):
        t = target.float().contiguous()
        _, elem, _ = _launch(pred_logits, t, None, None, 0, 0, self.alpha, self.gamma, 1.0, True, False)
        return elem.view_as(pred_logits)

    __call__ = forward


class _FocalSum(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, target, mask, cls_index, num_classes, hw, alpha, gamma):
        total, _, grad = _launch(logits, target, mask, cls_index, num_classes, hw, alpha, gamma, 1.0, False, True)
        ctx.save_for_backward(grad.view_as(logits))
        return total[0]

    @staticmethod
    def backward(ctx, g):
        (grad,) = ctx.saved_tensors
        return grad * g, None, None, None, None, None, None, None


def focal_loss_sum(pred_logits, target=None, mask=None, cls_index=None, alpha=0.25, gamma=2.0):
    """sum(mask * FocalLoss(pred_logits, target)) with the gradient produced in the same pass
    (== `(cls_mask * cls_criterion(cls_head, cls_target)).sum()`, odtk/model.py:196-199).
    Either a dense one-hot `target` (+ optional dense `mask`) or `cls_index` int32 [groups, H*W]
    for logits shaped [groups, classes, H*W] (-1 background, -2 ignored)."""
    if cls_index is not None:
        ncls, hw = pred_logits.shape[-2], pred_logits.shape[-1]
        return _FocalSum.apply(pred_logits, None, None, cls_index.int().contiguous(), ncls, hw, alpha, gamma)
    t = target.float().contiguous()
    m = mask.float().expand_as(t).contiguous() if mask is not None else None
    return _FocalSum.apply(pred_logits, t, m, None, 0, 0, alpha, gamma)


class SmoothL1Loss:
    'Smooth L1 Loss (reference: odtk/loss.py:20-31)'

    def __init__(self, beta=0.11):
        self.beta = beta

    def forward(self, pred, target):
        _, elem, _ = _launch_l1(pred, target, None, self.beta, 1.0, True, False)
        return elem.view_as(pred)

    __call__ = forward


def _launch_l1(pred, target, mask, beta, grad_scale, want_elem, want_grad):
    if not pred.is_cuda:
        raise RuntimeError("pred must be a CUDA tensor")
    L = _lib.lib()
    x, t = pred.float().contiguous(), target.float().contiguous()
    m = mask.float().expand_as(x).contiguous() if mask is not None else None
    elem = torch.empty_like(x) if want_elem else None
    grad = torch.empty_like(x) if want_grad else None
    total = torch.empty(1, dtype=torch.float32, device=x.device)

    def p(v):
        return ctypes.c_void_p(v.data_ptr()) if v is not None else None
    args = (p(x), p(t), p(m), x.numel(), float(beta), float(grad_scale), p(elem), p(total), p(grad))
    size = _lib.check(L.odtk_smooth_l1_loss(*args, None, 0, None), "smooth_l1 (workspace query)")
    ws = torch.empty(int(size), dtype=torch.uint8, device=x.device)
    _lib.check(L.odtk_smooth_l1_loss(*args, ctypes.c_void_p(ws.data_ptr()), size,
                                     ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "smooth_l1")
    return total, elem, grad


class _L1Sum(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, target, mask, beta):
        total, _, grad = _launch_l1(pred, target, mask, beta, 1.0, False, True)
        ctx.save_for_backward(grad.view_as(pred))
        return total[0]

    @staticmethod
    def backward(ctx, g):
        (grad,) = ctx.saved_tensors
        return grad * g, None, None, None


def smooth_l1_loss_sum(pred, target, mask=None, beta=0.11):
    """sum(mask * SmoothL1Loss(pred, target)) with its gradient in the same pass
    (== `(box_mask * box_criterion(box_head, box_target)).sum()`, odtk/model.py:201-205)."""
    return _L1Sum.apply(pred, target, mask, beta)


def retina_loss(cls_heads, box_heads, cls_indices, box_targets, num_classes, alpha=0.25, gamma=2.0, beta=0.11,
                with_grad=False):
    """Model._compute_loss (odtk/model.py:186-210) for ALL pyramid levels in ONE kernel launch (odtk_retina_loss):
    cls_heads[l] [B, A*C, H, W] raw logits, box_heads[l] [B, A*nbox, H, W], cls_indices[l] [B, A, H, W] int32 (class,
    -1 background, -2 ignored: box.snap_to_anchors_batch), box_targets[l] [B, A, nbox, H, W].
    Returns (cls_loss, box_loss) 0-dim tensors, both already divided by sum_l max(1, #foreground_l); with_grad=True also
    returns (cls_grads, box_grads): d cls_loss / d cls_heads[l] and d box_loss / d box_heads[l]."""
    nl = len(cls_heads)
    if not (nl == len(box_heads) == len(cls_indices) == len(box_targets)) or nl == 0:
        raise ValueError("one entry per pyramid level in every list")
    dev = cls_heads[0].device
    if not cls_heads[0].is_cuda:
        raise RuntimeError("retina_loss needs CUDA tensors: there is no CPU path")
    batch = cls_heads[0].shape[0]
    num_anchors = cls_indices[0].shape[1]
    nbox = box_targets[0].shape[2]
    keep, levels = [], (_lib.LossLevel * nl)()
    cls_grads, box_grads = [], []
    for l in range(nl):
        c, b = cls_heads[l].float().contiguous(), box_heads[l].float().contiguous()
        ci, bt = cls_indices[l].int().contiguous(), box_targets[l].float().contiguous()
        if c.shape[1] != num_anchors * num_classes or b.shape[1] != num_anchors * nbox or tuple(ci.shape[2:]) != tuple(c.shape[2:]):
            raise ValueError("level %d: head / target shapes do not agree" % l)
        keep += [c, b, ci, bt]
        levels[l].cls_logits, levels[l].box_pred = c.data_ptr(), b.data_ptr()
        levels[l].cls_index, levels[l].box_target = ci.data_ptr(), bt.data_ptr()
        if with_grad:
            cls_grads.append(torch.empty_like(c))
            box_grads.append(torch.empty_like(b))
            levels[l].cls_grad, levels[l].box_grad = cls_grads[-1].data_ptr(), box_grads[-1].data_ptr()
        levels[l].height, levels[l].width = c.shape[2], c.shape[3]
    out = torch.empty(4, dtype=torch.float32, device=dev)
    L = _lib.lib()
    args = (batch, nl, ctypes.cast(levels, ctypes.c_void_p), int(num_anchors), int(num_classes), int(nbox), float(alpha),
            float(gamma), float(beta), ctypes.c_void_p(out.data_ptr()))
    size = _lib.check(L.odtk_retina_loss(*args, None, 0, None), "retina_loss (workspace query)")
    ws = torch.empty(int(size), dtype=torch.uint8, device=dev)
    _lib.check(L.odtk_retina_loss(*args, ctypes.c_void_p(ws.data_ptr()), size,
                                  ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "retina_loss")
    if with_grad:
        return out[0], out[1], cls_grads, box_grads
    return out[0], out[1]
