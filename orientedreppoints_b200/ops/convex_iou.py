"""Mirror of mmdet/ops/iou/iou_wrapper.py (convex_giou :12-17, convex_iou :21-25, convex_overlaps :27-30): IoU between
the convex hull of each 9-point set and each quadrilateral, and the GIoU of aligned pairs with its gradient with respect
to the points (the training loss's operator, losses.py)."""
import torch

from .. import _lib
from .box_iou_rotated import _check_rows


def convex_iou(pred, target):
    """pred: [ex_num, 18] cuda float (x0,y0,...,x8,y8); target: [gt_num, 8] -> [ex_num, gt_num] on pred.device"""
    if not (torch.is_tensor(pred) and pred.is_cuda and torch.is_tensor(target) and target.is_cuda):
        raise TypeError('ex_boxes must be a CUDA tensor')          # convex_iou_kernel.cu:317-318 AT_ASSERTM
    ex_num, gt_num = pred.size(0), target.size(0)
    if ex_num == 0 or gt_num == 0:
        return pred.new_zeros((ex_num, gt_num), dtype=torch.float32)
    p = pred.detach().float().contiguous().reshape(ex_num, 18)
    t = target.detach().float().contiguous().reshape(gt_num, 8)
    out = torch.empty((ex_num, gt_num), dtype=torch.float32, device=pred.device)
    with torch.cuda.device(pred.device):
        _lib.check(_lib.lib().orp_convex_iou(_lib.ptr(p), ex_num, _lib.ptr(t), gt_num, _lib.ptr(out),
                                             _lib.current_stream_ptr()), "orp_convex_iou")
    return out


def convex_overlaps(gt_rbboxes, points):
    return convex_iou(points, gt_rbboxes).transpose(1, 0)


def convex_giou(pred, target):
    """pred: [N, 18] cuda float (x0,y0,...,x8,y8); target: [N, 8], aligned pairs -> (giou [N], grad [N, 18]) float32 on
    pred.device: views of one [N, 19] tensor, row i = [d giou_i / d pred_i | giou_i].  Nothing is read back to the host."""
    _check_rows("convex_giou pred", pred, 18)
    _check_rows("convex_giou target", target, 8)
    if pred.size(0) != target.size(0):
        raise ValueError("convex_giou: pred has %d rows, target %d; the pairs are aligned"   # :833 AT_ASSERTM
                         % (pred.size(0), target.size(0)))
    if not (pred.is_cuda and target.is_cuda):
        raise TypeError('ex_boxes must be a CUDA tensor')          # convex_giou_kernel.cu:831-832 AT_ASSERTM
    n = pred.size(0)
    out = torch.empty((n, 19), dtype=torch.float32, device=pred.device)
    if n > 0:
        p = pred.detach().float().contiguous()
        t = target.detach().float().contiguous()
        with torch.cuda.device(pred.device):
            _lib.check(_lib.lib().orp_convex_giou(_lib.ptr(p), _lib.ptr(t), n, _lib.ptr(out), _lib.current_stream_ptr()),
                       "orp_convex_giou")
    return out[:, -1], out[:, 0:-1]
