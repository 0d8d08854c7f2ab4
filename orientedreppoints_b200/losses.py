"""Mirror of mmdet/models/losses/iou_loss.py:63-128: the GIoU loss between the convex hull of a point set and its target
quadrilateral that the configs name for loss_rbox_init / loss_rbox_refine, over ops.convex_giou (one device call).

The reference's training semantics are kept as they are, odd parts included: the gradient is the operator's analytic
one, weighted, with every row that has an element > 1 replaced by 1e-6, scaled by -loss_weight / N and returned from
backward whatever the incoming gradient; GIoULoss.forward multiplies the loss by loss_weight a second time; avg_factor is
accepted and unused.  The row filter is a mask and torch.where instead of torch.nonzero and an index write (same values),
so GIoULossFuction.forward makes no host synchronisation."""
import torch
import torch.nn as nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from .models import LOSSES
from .ops.convex_iou import convex_giou


class GIoULossFuction(Function):
    @staticmethod
    def forward(ctx, pred, target, weight=None, reduction=None, avg_factor=None, loss_weight=1.0):
        ctx.save_for_backward(pred)

        convex_gious, grad = convex_giou(pred, target)
        loss = 1 - convex_gious
        if weight is not None:
            loss = loss * weight
            grad = grad * weight.reshape(-1, 1)
        if reduction == 'sum':
            loss = loss.sum()
        elif reduction == 'mean':
            loss = loss.mean()

        # _unvalid_grad_filter: a row with any element > 1 becomes eps
        eps = 1e-6
        grad = torch.where((grad > 1).any(1, keepdim=True), eps, grad)

        # _reduce_grad
        ctx.convex_points_grad = -grad / grad.size(0) * loss_weight
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, input=None):
        return ctx.convex_points_grad, None, None, None, None, None


convex_giou_loss = GIoULossFuction.apply


@LOSSES.register_module
class GIoULoss(nn.Module):
    def __init__(self, reduction='mean', loss_weight=1.0):
        super(GIoULoss, self).__init__()
        self.reduction = reduction
        self.loss_weight = loss_weight

    def forward(self, pred, target, weight=None, avg_factor=None, reduction_override=None, **kwargs):
        if weight is not None and not torch.any(weight > 0):
            return (pred * weight.unsqueeze(-1)).sum()
        assert reduction_override in (None, 'none', 'mean', 'sum')
        reduction = reduction_override if reduction_override else self.reduction
        return self.loss_weight * convex_giou_loss(pred, target, weight, reduction, avg_factor, self.loss_weight)
