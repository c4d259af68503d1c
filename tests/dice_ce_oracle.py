"""monai.losses.DiceCELoss restated in torch ops (any dtype, any device) and its closed-form logit gradient.

Test and measurement infrastructure only: the package never imports it.  ``dice_ce_loss`` follows MONAI's published
definition: ``lambda_dice * DiceLoss(...) + lambda_ce * CE``, CE on the raw logits (cross-entropy over channels for C > 1,
BCEWithLogits for C == 1), ``include_background`` dropping channel 0 of the Dice only.  One addition: a label outside
[0, C) is an all-zero target row (MONAI leaves it undefined).  ``dice_ce_grad`` is d(loss)/d(logits) written out by hand --
the expression the backward kernel evaluates.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def dice_ce_target(logits: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
    """The target as a [N,C,...] tensor of logits' dtype: a [N,1,...] label map (C > 1) becomes one-hot rows, all zero where the
    label is outside [0, C); anything else is cast."""
    c = logits.shape[1]
    if c > 1 and target.shape[1] == 1:
        lab = target[:, 0].long()
        valid = ((lab >= 0) & (lab < c)).unsqueeze(1).to(logits.dtype)
        return F.one_hot(lab.clamp(0, c - 1), c).movedim(-1, 1).to(logits.dtype) * valid
    return target.to(logits.dtype)


def _act(logits, sigmoid, softmax):
    if sigmoid:
        return torch.sigmoid(logits)
    if softmax and logits.shape[1] > 1:
        return torch.softmax(logits, dim=1)
    return logits


def dice_ce_loss(logits: torch.Tensor, target: torch.Tensor, *, include_background: bool = True, sigmoid: bool = False,
                 softmax: bool = False, squared_pred: bool = False, jaccard: bool = False, batch: bool = False,
                 reduction: str = "mean", smooth_nr: float = 1e-5, smooth_dr: float = 1e-5, lambda_dice: float = 1.0,
                 lambda_ce: float = 1.0, to_onehot_y: bool = True) -> torch.Tensor:
    """``to_onehot_y`` is accepted for MONAI's call signature; the target's channel count decides (a [N,1,...] target with C > 1
    is a label map)."""
    del to_onehot_y
    c = logits.shape[1]
    t = dice_ce_target(logits, target)
    p = _act(logits, sigmoid, softmax)
    pd, td = (p[:, 1:], t[:, 1:]) if (not include_background and c > 1) else (p, t)
    axes = list(range(2, p.dim()))
    if batch:
        axes = [0] + axes
    inter = (pd * td).sum(dim=axes)
    ground = (td * td).sum(dim=axes) if squared_pred else td.sum(dim=axes)
    pred = (pd * pd).sum(dim=axes) if squared_pred else pd.sum(dim=axes)
    denom = ground + pred
    if jaccard:
        denom = 2.0 * (denom - inter)
    f = 1.0 - (2.0 * inter + smooth_nr) / (denom + smooth_dr)
    if c > 1:
        ce = -(t * torch.log_softmax(logits, dim=1)).sum()
    else:
        ce = F.binary_cross_entropy_with_logits(logits, t, reduction="sum")
    voxels = logits.shape[0] * logits[0, 0].numel()
    if reduction == "mean":
        return lambda_dice * f.mean() + lambda_ce * ce / voxels
    return lambda_dice * f.sum() + lambda_ce * ce


def dice_ce_grad(logits: torch.Tensor, target: torch.Tensor, *, include_background: bool = True, sigmoid: bool = False,
                 softmax: bool = False, squared_pred: bool = False, jaccard: bool = False, batch: bool = False,
                 reduction: str = "mean", smooth_nr: float = 1e-5, smooth_dr: float = 1e-5, lambda_dice: float = 1.0,
                 lambda_ce: float = 1.0, to_onehot_y: bool = True) -> torch.Tensor:
    """Closed-form d(dice_ce_loss)/d(logits):
        g_c  = w * (dF/dI t_c + dF/dP dP/dp_c)    F = 1 - (2I + nr) / (Den + dr), D' = Den + dr
               plain Den = P + T:         dF/dI = -2/D',                  dF/dP = (2I + nr)/D'^2
               jaccard Den = 2(P + T - I): dF/dI = -2/D' - 2(2I + nr)/D'^2, dF/dP = 2(2I + nr)/D'^2
               w = lambda_dice / (number of Dice terms) for mean, lambda_dice for sum; 0 on a dropped background channel
        dx_c = p_c (g_c - sum_k p_k g_k)  [softmax],  g_c p_c (1 - p_c)  [sigmoid],  g_c  [identity]
             + s (q_c sum_k t_k - t_c)    [C > 1, q = softmax],  s (sigmoid(x) - t)  [C == 1]
               s = lambda_ce / (N * S) for mean, lambda_ce for sum"""
    del to_onehot_y
    n, c = logits.shape[:2]
    t = dice_ce_target(logits, target)
    p = _act(logits, sigmoid, softmax)
    axes = list(range(2, p.dim()))
    if batch:
        axes = [0] + axes
    inter = (p * t).sum(dim=axes, keepdim=True)
    ground = (t * t).sum(dim=axes, keepdim=True) if squared_pred else t.sum(dim=axes, keepdim=True)
    pred = (p * p).sum(dim=axes, keepdim=True) if squared_pred else p.sum(dim=axes, keepdim=True)
    den = ground + pred
    if jaccard:
        den = 2.0 * (den - inter)
    d = den + smooth_dr
    num = 2.0 * inter + smooth_nr
    if jaccard:
        dfdi, dfdp = -2.0 / d - 2.0 * num / (d * d), 2.0 * num / (d * d)
    else:
        dfdi, dfdp = -2.0 / d, num / (d * d)
    c_lo = 1 if (not include_background and c > 1) else 0
    terms = (1 if batch else n) * (c - c_lo)
    w = torch.full((1, c) + (1,) * (p.dim() - 2), lambda_dice / terms if reduction == "mean" else lambda_dice,
                   dtype=logits.dtype, device=logits.device)
    w[:, :c_lo] = 0.0
    g = w * (dfdi * t + dfdp * (2.0 * p if squared_pred else 1.0))
    if softmax and c > 1:
        dx = p * (g - (p * g).sum(dim=1, keepdim=True))
    elif sigmoid:
        dx = g * p * (1.0 - p)
    else:
        dx = g
    s = lambda_ce / (n * logits[0, 0].numel()) if reduction == "mean" else lambda_ce
    if c > 1:
        dx = dx + s * (torch.softmax(logits, dim=1) * t.sum(dim=1, keepdim=True) - t)
    else:
        dx = dx + s * (torch.sigmoid(logits) - t)
    return dx
