"""ORACLE / TEST INFRASTRUCTURE ONLY. Minimal stand-in for the un-vendored dependency named by the
package path (mmcv-full==1.5.3 / mmdet==2.25.0, environment.yml:27-28); restates only the
symbols imported at team_code_transfuser/model.py:20-30. parity unpinned (source absent)."""
import torch
import torch.nn.functional as F
from torch import nn


def _reduce(loss, weight, reduction, avg_factor):
    """mmdet weight_reduce_loss: elementwise * weight, then mean / sum / (sum / avg_factor)."""
    if weight is not None:
        loss = loss * weight
    if avg_factor is None:
        if reduction == 'mean':
            return loss.mean()
        if reduction == 'sum':
            return loss.sum()
        return loss
    if reduction == 'mean':
        return loss.sum() / avg_factor
    if reduction == 'none':
        return loss
    raise ValueError('avg_factor can not be used with reduction="sum"')


class _Loss(nn.Module):
    def __init__(self, reduction='mean', loss_weight=1.0, **kw):
        super().__init__()
        self.reduction = reduction
        self.loss_weight = loss_weight
        self.kw = kw

    def forward(self, pred, target, weight=None, avg_factor=None, reduction_override=None):
        reduction = reduction_override if reduction_override else self.reduction
        return self.loss_weight * _reduce(self.elementwise(pred, target), weight, reduction, avg_factor)


class L1Loss(_Loss):
    def elementwise(self, pred, target):
        return torch.abs(pred - target)


class SmoothL1Loss(_Loss):
    def elementwise(self, pred, target):
        beta = self.kw.get('beta', 1.0)
        diff = torch.abs(pred - target)
        return torch.where(diff < beta, 0.5 * diff * diff / beta, diff - 0.5 * beta)


class GaussianFocalLoss(_Loss):
    def elementwise(self, pred, target):
        alpha, gamma, eps = self.kw.get('alpha', 2.0), self.kw.get('gamma', 4.0), 1e-12
        pos_weights = target.eq(1)
        neg_weights = (1 - target).pow(gamma)
        pos_loss = -(pred + eps).log() * (1 - pred).pow(alpha) * pos_weights
        neg_loss = -(1 - pred + eps).log() * pred.pow(alpha) * neg_weights
        return pos_loss + neg_loss


class CrossEntropyLoss(_Loss):
    def forward(self, cls_score, label, weight=None, avg_factor=None, reduction_override=None, **kwargs):
        reduction = reduction_override if reduction_override else self.reduction
        loss = F.cross_entropy(cls_score, label, weight=None, reduction='none', ignore_index=-100)
        if weight is not None:
            weight = weight.float()
        return self.loss_weight * _reduce(loss, weight, reduction, avg_factor)


_LOSSES = dict(L1Loss=L1Loss, SmoothL1Loss=SmoothL1Loss, GaussianFocalLoss=GaussianFocalLoss,
               CrossEntropyLoss=CrossEntropyLoss)


def build_loss(cfg):
    cfg = dict(cfg)
    return _LOSSES[cfg.pop('type')](**cfg)
