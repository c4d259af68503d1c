"""monai.losses.FocalLoss, DiceFocalLoss, TverskyLoss and GeneralizedDiceLoss restated in torch ops (any dtype, any device), and
the closed-form logit gradients the fused kernels evaluate.

Test and measurement infrastructure only: the package never imports it.  MONAI's published definitions, restated:

Shared steps: the activation, then ``to_onehot_y`` (here: a [N,1,...] target with C > 1 is a label map and becomes one-hot rows,
all zero for a label outside [0, C) -- ``dice_ce_oracle.dice_ce_target``), then ``include_background=False`` drops channel 0
(ignored with C == 1).  ``reduction`` is "mean" or "sum".

- FocalLoss(include_background, gamma, alpha, weight, reduction, use_softmax).  The background is dropped *before* the activation.
  Sigmoid form, per element: ``(x - x t - logsigmoid(x)) exp(gamma logsigmoid(-x (2t - 1)))``, times ``t alpha + (1 - t)(1 - alpha)``
  with alpha.  Softmax form: ``ls = log_softmax(x)`` over the kept channels, ``-(1 - exp(ls))^gamma ls t``, times the per-channel
  ``[1 - alpha, alpha, alpha, ...]`` with alpha -- which MONAI ignores (with a warning) when the background is dropped.
  ``weight``: a scalar or C' per-class factors >= 0, applied when C' > 1.  "mean" divides the total by N C' S; "sum" takes the
  mean over the voxels of each (n, c) and sums those (MONAI's FocalLoss does so for backward compatibility).
- DiceFocalLoss: ``lambda_dice DiceLoss(...) + lambda_focal FocalLoss(..., use_softmax=softmax)``, one-hot conversion once.  Under
  softmax with the background dropped the Dice takes its softmax over all C channels, the focal term over channels 1..C-1.
- TverskyLoss: per (n, c), per c with batch, ``f = 1 - (I + nr) / (I + alpha (P - I) + beta (T - I) + dr)`` with I = sum p t,
  P = sum p, T = sum t (MONAI's fp = alpha sum p (1 - t), fn = beta sum (1 - p) t).
- GeneralizedDiceLoss: ``w_c = 1/T_c^2, 1/T_c or 1``; infinite weights become 0, then get the largest weight added (per sample,
  or over everything with batch); ``f = 1 - (2 sum_c w_c I_c + nr) / (sum_c w_c (P_c + T_c) + dr)`` per n, or once with batch.
  The weights carry no gradient.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from dice_ce_oracle import dice_ce_target

W_TYPES = ("square", "simple", "uniform")


def _act(logits, sigmoid, softmax):
    if sigmoid:
        return torch.sigmoid(logits)
    if softmax and logits.shape[1] > 1:
        return torch.softmax(logits, dim=1)
    return logits


def _lo(c, include_background):
    return 1 if (not include_background and c > 1) else 0


def _reduce(f, reduction):
    return f.mean() if reduction == "mean" else f.sum()


def _focal_alpha(alpha, use_softmax, include_background):
    return None if (use_softmax and not include_background) else alpha


def _class_factors(kept, weight, like):
    """[1, C', 1, ...] factors (ones without weights or with one kept channel)"""
    shape = (1, kept) + (1,) * (like.dim() - 2)
    if weight is None or kept == 1:
        return torch.ones(shape, dtype=like.dtype, device=like.device)
    w = torch.as_tensor(weight, dtype=like.dtype).to(like.device).reshape(-1)
    if w.numel() == 1:
        w = w.expand(kept)
    return w.reshape(shape)


def focal_elements(logits, t, *, include_background=True, gamma=2.0, alpha=None, weight=None, use_softmax=False):
    """the per-element focal terms [N, C', ...] on the kept channels, class factors applied"""
    lo = _lo(logits.shape[1], include_background)
    x, t = logits[:, lo:], t[:, lo:]
    alpha = _focal_alpha(alpha, use_softmax, include_background)
    if use_softmax:
        ls = torch.log_softmax(x, dim=1)
        loss = -(1 - ls.exp()).pow(gamma) * ls * t
        if alpha is not None:
            fac = torch.tensor([1 - alpha] + [alpha] * (t.shape[1] - 1), dtype=x.dtype, device=x.device)
            loss = fac.view((1, -1) + (1,) * (x.dim() - 2)) * loss
    else:
        loss = x - x * t - F.logsigmoid(x)
        loss = (F.logsigmoid(-x * (t * 2 - 1)) * gamma).exp() * loss
        if alpha is not None:
            loss = (t * alpha + (1 - t) * (1 - alpha)) * loss
    return _class_factors(x.shape[1], weight, x) * loss


def focal_loss(logits, target, *, include_background=True, gamma=2.0, alpha=None, weight=None, reduction="mean",
               use_softmax=False, to_onehot_y=True):
    del to_onehot_y
    t = dice_ce_target(logits, target)
    loss = focal_elements(logits, t, include_background=include_background, gamma=gamma, alpha=alpha, weight=weight,
                          use_softmax=use_softmax)
    if reduction == "sum":
        return loss.mean(dim=list(range(2, loss.dim()))).sum()
    return loss.mean()


def overlap_sums(p, t, include_background, batch):
    """(I, P, T) over the kept channels: [N, C'] or, with batch, [C']"""
    lo = _lo(p.shape[1], include_background)
    p, t = p[:, lo:], t[:, lo:]
    axes = list(range(2, p.dim()))
    if batch:
        axes = [0] + axes
    return (p * t).sum(dim=axes), p.sum(dim=axes), t.sum(dim=axes)


def dice_f(p, t, *, include_background=True, squared_pred=False, jaccard=False, batch=False, smooth_nr=1e-5, smooth_dr=1e-5):
    lo = _lo(p.shape[1], include_background)
    pd, td = p[:, lo:], t[:, lo:]
    axes = list(range(2, p.dim()))
    if batch:
        axes = [0] + axes
    inter = (pd * td).sum(dim=axes)
    ground = (td * td).sum(dim=axes) if squared_pred else td.sum(dim=axes)
    pred = (pd * pd).sum(dim=axes) if squared_pred else pd.sum(dim=axes)
    denom = ground + pred
    if jaccard:
        denom = 2.0 * (denom - inter)
    return 1.0 - (2.0 * inter + smooth_nr) / (denom + smooth_dr)


def tversky_f(p, t, *, include_background=True, alpha=0.5, beta=0.5, batch=False, smooth_nr=1e-5, smooth_dr=1e-5):
    lo = _lo(p.shape[1], include_background)
    p0, g0 = p[:, lo:], t[:, lo:]
    p1, g1 = 1 - p0, 1 - g0
    axes = list(range(2, p.dim()))
    if batch:
        axes = [0] + axes
    tp = (p0 * g0).sum(dim=axes)
    fp = alpha * (p0 * g1).sum(dim=axes)
    fn = beta * (p1 * g0).sum(dim=axes)
    return 1.0 - (tp + smooth_nr) / (tp + fp + fn + smooth_dr)


def gdice_weights(T, w_type, batch):
    """weights from the target sums T ([N, C'] or [C'] with batch), infinite ones replaced as MONAI does"""
    T = T.detach()
    w = {"square": lambda g: torch.reciprocal(g * g), "simple": torch.reciprocal, "uniform": torch.ones_like}[w_type](T)
    infs = torch.isinf(w)
    w = torch.where(infs, torch.zeros_like(w), w)
    if batch:
        return w + infs * torch.max(w)
    return w + infs * torch.max(w, dim=1, keepdim=True)[0]


def gdice_f(p, t, *, include_background=True, w_type="square", batch=False, smooth_nr=1e-5, smooth_dr=1e-5):
    inter, pred, ground = overlap_sums(p, t, include_background, batch)
    w = gdice_weights(ground, w_type, batch)
    dim = 0 if batch else 1
    numer = 2.0 * (inter * w).sum(dim) + smooth_nr
    denom = ((ground + pred) * w).sum(dim) + smooth_dr
    return 1.0 - numer / denom


def tversky_loss(logits, target, *, include_background=True, sigmoid=False, softmax=False, alpha=0.5, beta=0.5, reduction="mean",
                 smooth_nr=1e-5, smooth_dr=1e-5, batch=False, to_onehot_y=True):
    del to_onehot_y
    t = dice_ce_target(logits, target)
    return _reduce(tversky_f(_act(logits, sigmoid, softmax), t, include_background=include_background, alpha=alpha, beta=beta,
                             batch=batch, smooth_nr=smooth_nr, smooth_dr=smooth_dr), reduction)


def generalized_dice_loss(logits, target, *, include_background=True, sigmoid=False, softmax=False, w_type="square",
                          reduction="mean", smooth_nr=1e-5, smooth_dr=1e-5, batch=False, to_onehot_y=True):
    del to_onehot_y
    t = dice_ce_target(logits, target)
    return _reduce(gdice_f(_act(logits, sigmoid, softmax), t, include_background=include_background, w_type=w_type, batch=batch,
                           smooth_nr=smooth_nr, smooth_dr=smooth_dr), reduction)


def dice_focal_loss(logits, target, *, include_background=True, sigmoid=False, softmax=False, squared_pred=False, jaccard=False,
                    reduction="mean", smooth_nr=1e-5, smooth_dr=1e-5, batch=False, gamma=2.0, lambda_dice=1.0, lambda_focal=1.0,
                    alpha=None, to_onehot_y=True):
    del to_onehot_y
    t = dice_ce_target(logits, target)
    dice = _reduce(dice_f(_act(logits, sigmoid, softmax), t, include_background=include_background, squared_pred=squared_pred,
                          jaccard=jaccard, batch=batch, smooth_nr=smooth_nr, smooth_dr=smooth_dr), reduction)
    focal = focal_loss(logits, t, include_background=include_background, gamma=gamma, alpha=alpha, reduction=reduction,
                       use_softmax=softmax)
    return lambda_dice * dice + lambda_focal * focal


# ------------------------------------------------------------------------------------------------ closed-form gradients
def _pooled(v, batch, n):
    return v.sum(dim=0, keepdim=True).expand(n, *v.shape[1:]) if batch else v


def overlap_coef(p, t, *, kind="dice", include_background=True, squared_pred=False, jaccard=False, batch=False, smooth_nr=1e-5,
                 smooth_dr=1e-5, alpha=0.5, beta=0.5, w_type="square", reduction="mean", lam=1.0):
    """(a, b) [N, C] with d(lam * reduced f)/dp_c = a t_c + b dP/dp_c -- the finalize's coefficients, 0 on a dropped channel:
        Dice     F = 1 - (2I+nr)/D', D' = Den + dr: dF/dI = -2/D' (- 2(2I+nr)/D'^2 jaccard), dF/dP = (2I+nr)/D'^2 (x2 jaccard)
        Tversky  F = 1 - (I+nr)/D', D' = I + a(P-I) + b(T-I) + dr: dF/dI = -1/D' + (I+nr)(1-a-b)/D'^2, dF/dP = a(I+nr)/D'^2
        GDice    F = 1 - A/B per group: dF/dI_c = -2 w_c / B, dF/dP_c = A w_c / B^2"""
    n, c = p.shape[:2]
    lo = _lo(c, include_background)
    axes = list(range(2, p.dim()))
    I = (p * t).sum(dim=axes)
    P = (p * p).sum(dim=axes) if squared_pred else p.sum(dim=axes)
    T = (t * t).sum(dim=axes) if squared_pred else t.sum(dim=axes)
    I, P, T = _pooled(I, batch, n), _pooled(P, batch, n), _pooled(T, batch, n)
    if kind == "gdice":
        groups = 1 if batch else n
        w = gdice_weights(T[:, lo:] if not batch else T[:1, lo:], w_type, False)
        w = w.expand(n, -1) if batch else w
        A = 2.0 * (w * I[:, lo:]).sum(dim=1, keepdim=True) + smooth_nr
        B = (w * (P[:, lo:] + T[:, lo:])).sum(dim=1, keepdim=True) + smooth_dr
        scale = lam / groups if reduction == "mean" else lam
        a = torch.zeros_like(I)
        b = torch.zeros_like(I)
        a[:, lo:] = scale * (-2.0 * w / B)
        b[:, lo:] = scale * (A * w / (B * B))
        return a, b
    if kind == "tversky":
        D = I + alpha * (P - I) + beta * (T - I) + smooth_dr
        num = I + smooth_nr
        dfdi, dfdp = -1.0 / D + num * (1.0 - alpha - beta) / (D * D), alpha * num / (D * D)
    else:
        den = P + T
        if jaccard:
            den = 2.0 * (den - I)
        D = den + smooth_dr
        num = 2.0 * I + smooth_nr
        if jaccard:
            dfdi, dfdp = -2.0 / D - 2.0 * num / (D * D), 2.0 * num / (D * D)
        else:
            dfdi, dfdp = -2.0 / D, num / (D * D)
    terms = (1 if batch else n) * (c - lo)
    w = torch.full((1, c), lam / terms if reduction == "mean" else lam, dtype=p.dtype, device=p.device)
    w[:, :lo] = 0.0
    return w * dfdi, w * dfdp


def act_backward(logits, p, g, sigmoid, softmax):
    """d/dx of sum_c g_c p_c with p = act(x), g held fixed"""
    if softmax and logits.shape[1] > 1:
        return p * (g - (p * g).sum(dim=1, keepdim=True))
    if sigmoid:
        return g * p * (1.0 - p)
    return g


def focal_grad(logits, t, *, include_background=True, gamma=2.0, alpha=None, weight=None, use_softmax=False):
    """d(sum of the focal elements)/d(logits), zero on a dropped channel:
        sigmoid  a E [(sigmoid(x) - t) - gamma s l0 sigmoid(x s)],  s = 2t - 1, l0 = x - x t - logsigmoid(x),
                 E = exp(gamma logsigmoid(-x s)), a = class factor (times t alpha + (1 - t)(1 - alpha))
        softmax  u_j - p'_j sum_c u_c,  u_c = -a_c t_c [(1 - p'_c)^gamma - gamma (1 - p'_c)^(gamma - 1) p'_c ls_c]"""
    c = logits.shape[1]
    lo = _lo(c, include_background)
    x, tt = logits[:, lo:], t[:, lo:]
    a = _class_factors(x.shape[1], weight, x)
    alpha = _focal_alpha(alpha, use_softmax, include_background)
    out = torch.zeros_like(logits)
    if use_softmax:
        if alpha is not None:
            fac = torch.tensor([1 - alpha] + [alpha] * (x.shape[1] - 1), dtype=x.dtype, device=x.device)
            a = a * fac.view((1, -1) + (1,) * (x.dim() - 2))
        ls = torch.log_softmax(x, dim=1)
        p = ls.exp()
        omp = 1 - p
        pw = omp.pow(gamma)
        d = gamma * omp.pow(gamma - 1) * p * ls if gamma != 0 else torch.zeros_like(ls)
        d = torch.where(omp > 0, d, torch.zeros_like(d))
        u = -a * tt * (pw - d)
        out[:, lo:] = u - p * u.sum(dim=1, keepdim=True)
    else:
        s = 2 * tt - 1
        l0 = x - x * tt - F.logsigmoid(x)
        E = (F.logsigmoid(-x * s) * gamma).exp()
        if alpha is not None:
            a = a * (tt * alpha + (1 - tt) * (1 - alpha))
        out[:, lo:] = a * E * ((torch.sigmoid(x) - tt) - gamma * s * l0 * torch.sigmoid(x * s))
    return out


def fused_grad(logits, target, *, kind="dice", act=None, include_background=True, squared_pred=False, jaccard=False, batch=False,
               reduction="mean", smooth_nr=1e-5, smooth_dr=1e-5, alpha=0.5, beta=0.5, w_type="square", lambda_dice=1.0,
               lambda_focal=0.0, gamma=2.0, focal_alpha=None, weight=None, focal_softmax=False):
    """closed-form d/d(logits) of lambda_dice * overlap + lambda_focal * focal, the expression the backward kernel evaluates"""
    n, c = logits.shape[:2]
    t = dice_ce_target(logits, target)
    p = _act(logits, act == "sigmoid", act == "softmax")
    dx = torch.zeros_like(logits)
    if lambda_dice != 0:
        a, b = overlap_coef(p, t, kind=kind, include_background=include_background, squared_pred=squared_pred, jaccard=jaccard,
                            batch=batch, smooth_nr=smooth_nr, smooth_dr=smooth_dr, alpha=alpha, beta=beta, w_type=w_type,
                            reduction=reduction, lam=lambda_dice)
        shape = (n, c) + (1,) * (p.dim() - 2)
        g = a.reshape(shape) * t + b.reshape(shape) * (2.0 * p if squared_pred else 1.0)
        dx = act_backward(logits, p, g, act == "sigmoid", act == "softmax")
    if lambda_focal != 0:
        kept = c - _lo(c, include_background)
        S = logits[0, 0].numel()
        scale = lambda_focal / (n * kept * S) if reduction == "mean" else lambda_focal / S
        dx = dx + scale * focal_grad(logits, t, include_background=include_background, gamma=gamma, alpha=focal_alpha, weight=weight,
                                     use_softmax=focal_softmax)
    return dx
