"""The reference's training criterion on the device: same classes, constructor arguments and forward signatures as
TaskPrompter/losses/loss_functions.py and loss_schemes.py (InvPT's are identical), so `get_criterion(p)`-style code
only swaps the import. Every loss value is ONE float tensor on the GPU produced by libmtt_sm90.so reductions
(mtt_loss_*), with no host synchronisation, and is differentiable with respect to the prediction through a custom
autograd.Function whose backward is the matching mtt_loss_*_grad kernel -- the scalar and the first gradient of the
training step of TP/utils/train_utils.py:34-51 (SURVEY.md section 8f N3; the backward of the model itself is N1).
"""
import ctypes as C

import torch
import torch.nn as nn

from . import lib as _L
from .ops import _launch, _ptr


def _ws(device):
    return torch.zeros(int(_L.load().mtt_loss_workspace_bytes()) // 8, dtype=torch.float64, device=device)


def _prep(out, label):
    if not out.is_cuda:
        raise RuntimeError("mtt_b200 losses have no CPU path: predictions must be CUDA tensors")
    return out.detach().float().contiguous(), label.detach().to(device=out.device, dtype=torch.float32).contiguous()


class _CE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, out, label, ignore_index, balanced):
        x, y = _prep(out, label)
        B, Cc, H, W = x.shape
        assert y.numel() == B * H * W, "label must be [B,1,H,W]"
        loss, ws = torch.empty((), device=x.device), _ws(x.device)
        _launch("mtt_loss_cross_entropy", _ptr(x), _ptr(y), B, Cc, H, W, float(ignore_index), int(balanced), _ptr(loss),
                _ptr(ws))
        ctx.save_for_backward(x, y, ws)
        ctx.args = (float(ignore_index), int(balanced), out.dtype)
        return loss

    @staticmethod
    def backward(ctx, g):
        x, y, ws = ctx.saved_tensors
        B, Cc, H, W = x.shape
        d = torch.empty_like(x)
        gs = g.detach().float().contiguous()
        _launch("mtt_loss_cross_entropy_grad", _ptr(x), _ptr(y), B, Cc, H, W, ctx.args[0], ctx.args[1], _ptr(gs),
                _ptr(d), _ptr(ws))
        return d.to(ctx.args[2]), None, None, None


class _BCE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, out, label, ignore_index, pos_weight):
        x, y = _prep(out, label)
        assert x.numel() == y.numel()
        hed = pos_weight is None
        loss, ws = torch.empty((), device=x.device), _ws(x.device)
        _launch("mtt_loss_balanced_bce", _ptr(x), _ptr(y), x.numel(), float(ignore_index),
                0.0 if hed else float(pos_weight), int(hed), _ptr(loss), _ptr(ws))
        ctx.save_for_backward(x, y, ws)
        ctx.args = (float(ignore_index), 0.0 if hed else float(pos_weight), int(hed), out.dtype)
        return loss

    @staticmethod
    def backward(ctx, g):
        x, y, ws = ctx.saved_tensors
        d = torch.empty_like(x)
        gs = g.detach().float().contiguous()
        _launch("mtt_loss_balanced_bce_grad", _ptr(x), _ptr(y), x.numel(), ctx.args[0], ctx.args[1], ctx.args[2],
                _ptr(gs), _ptr(d), _ptr(ws))
        return d.to(ctx.args[3]), None, None, None


class _L1(torch.autograd.Function):
    @staticmethod
    def forward(ctx, out, label, ignore_index, use_ignore, normalize):
        x, y = _prep(out, label)
        B, Cc, H, W = x.shape
        assert tuple(y.shape) == tuple(x.shape)
        loss, ws = torch.empty((), device=x.device), _ws(x.device)
        _launch("mtt_loss_l1", _ptr(x), _ptr(y), B, Cc, H, W, float(ignore_index), int(use_ignore), int(normalize),
                _ptr(loss), _ptr(ws))
        ctx.save_for_backward(x, y, ws)
        ctx.args = (float(ignore_index), int(use_ignore), int(normalize), out.dtype)
        return loss

    @staticmethod
    def backward(ctx, g):
        x, y, ws = ctx.saved_tensors
        B, Cc, H, W = x.shape
        d = torch.empty_like(x)
        gs = g.detach().float().contiguous()
        _launch("mtt_loss_l1_grad", _ptr(x), _ptr(y), B, Cc, H, W, ctx.args[0], ctx.args[1], ctx.args[2], _ptr(gs),
                _ptr(d), _ptr(ws))
        return d.to(ctx.args[3]), None, None, None, None


class CrossEntropyLoss(nn.Module):
    """loss_functions.py:15-55: cross entropy with ignore regions (reduction 'mean': sum / max(n_valid, 1));
    balanced=True: binary class weights (1 - w_pos, w_pos), w_pos = share of negative labels."""

    def __init__(self, ignore_index=255, class_weight=None, balanced=False):
        super().__init__()
        if class_weight is not None:
            raise NotImplementedError("mtt_b200 CrossEntropyLoss: fixed class_weight is not used by any reference config")
        self.ignore_index, self.balanced = ignore_index, balanced

    def forward(self, out, label, reduction='mean'):
        if reduction != 'mean':
            raise NotImplementedError("mtt_b200 losses implement the reduction the training loop uses ('mean')")
        return _CE.apply(out, label, self.ignore_index, self.balanced)


class BalancedBinaryCrossEntropyLoss(nn.Module):
    """loss_functions.py:57-87."""

    def __init__(self, pos_weight=None, ignore_index=255):
        super().__init__()
        self.pos_weight, self.ignore_index = pos_weight, ignore_index

    def forward(self, output, label, reduction='mean'):
        if reduction != 'mean':
            raise NotImplementedError("mtt_b200 losses implement the reduction the training loop uses ('mean')")
        return _BCE.apply(output, label, self.ignore_index, self.pos_weight)


class L1Loss(nn.Module):
    """loss_functions.py:144-176."""

    def __init__(self, normalize=False, ignore_index=0, ignore_invalid_area=True):
        super().__init__()
        self.normalize, self.ignore_invalid_area, self.ignore_index = normalize, ignore_invalid_area, ignore_index

    def forward(self, out, label, reduction='mean'):
        if reduction != 'mean':
            raise NotImplementedError("mtt_b200 losses implement the reduction the training loop uses ('mean')")
        return _L1.apply(out, label, self.ignore_index, self.ignore_invalid_area, self.normalize)


class MultiTaskLoss(nn.Module):
    """loss_schemes.py:8-39: {task: loss_t, 'total': sum_t w_t loss_t} (all scalars stay on the device)."""

    def __init__(self, p, tasks, loss_ft, loss_weights):
        super().__init__()
        assert set(tasks) == set(loss_ft.keys()) == set(loss_weights.keys())
        if '3ddet' in tasks:
            raise NotImplementedError("mtt_b200: the 3D-detection loss needs mmdet3d (SURVEY.md 8f N4)")
        self.p, self.tasks, self.loss_ft, self.loss_weights = p, list(tasks), loss_ft, loss_weights

    def forward(self, pred, gt, tasks):
        out = {t: self.loss_ft[t](pred[t], gt[t]) for t in tasks}
        out['total'] = torch.sum(torch.stack([self.loss_weights[t] * out[t] for t in tasks]))
        return out


def get_loss(p, task=None):
    """utils/common_config.py:211-237."""
    if task == 'edge':
        return BalancedBinaryCrossEntropyLoss(pos_weight=p['edge_w'], ignore_index=p['ignore_index'])
    if task in ('semseg', 'human_parts'):
        return CrossEntropyLoss(ignore_index=p['ignore_index'])
    if task == 'normals':
        return L1Loss(normalize=True, ignore_index=p['ignore_index'])
    if task == 'sal':
        return CrossEntropyLoss(balanced=True, ignore_index=p['ignore_index'])
    if task == 'depth':
        return L1Loss(ignore_invalid_area=p['ignore_invalid_area_depth'], ignore_index=-1)
    return None


def get_criterion(p):
    """utils/common_config.py:240-244."""
    names = list(p['TASKS']['NAMES'])
    loss_ft = nn.ModuleDict({t: get_loss(p, t) for t in names})
    return MultiTaskLoss(p, names, loss_ft, p['loss_kwargs']['loss_weights'])
