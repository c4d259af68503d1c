"""monai.losses.HausdorffDTLoss and LogHausdorffDTLoss restated in torch fp64, with scipy.ndimage.distance_transform_edt for the
distance fields, and a brute-force field to check that restatement.

Test and measurement infrastructure only: the package never imports it.  MONAI's published definition, restated:

- ``p = act(input)``: sigmoid, softmax over the channels (ignored with C == 1), or identity.  ``to_onehot_y`` (here: a [N,1,...]
  target with C > 1 is a label map and becomes one-hot rows, all zero for a label outside [0, C) -- ``dice_ce_target``), then
  ``include_background=False`` drops channel 0 of both (ignored with C == 1).
- For every kept channel c and sample n the distance field of a mask ``m = img > 0.5`` is ``edt(m) + edt(~m)`` when m is neither
  empty nor full, else 0; MONAI stores it in a float32 tensor, so each term is scipy's fp64 distance rounded to fp32.  The
  fields of the prediction (from the detached p) and of the target carry no gradient.
- ``f_c = mean over the voxels (and over n with batch) of (p_c - t_c)^2 (pdt_c^alpha + tdt_c^alpha)``; the loss is the mean or
  sum of all f terms.  ``LogHausdorffDTLoss`` is ``log(HausdorffDTLoss + 1)``.
"""
from __future__ import annotations

import numpy as np
import torch
from scipy.ndimage import distance_transform_edt

from dice_ce_oracle import dice_ce_target


def mask_field(mask: np.ndarray) -> np.ndarray:
    """fp32 edt(mask) + edt(~mask) of one boolean volume, 0 when the mask is empty or full"""
    mask = np.asarray(mask, dtype=bool)
    if not mask.any() or mask.all():
        return np.zeros(mask.shape, dtype=np.float32)
    return distance_transform_edt(mask).astype(np.float32) + distance_transform_edt(~mask).astype(np.float32)


def brute_field(mask: np.ndarray) -> np.ndarray:
    """the same field from every pair of voxels: the distance to the nearest voxel of the other value, in fp64, rounded to fp32"""
    mask = np.asarray(mask, dtype=bool)
    out = np.zeros(mask.shape, dtype=np.float32)
    if not mask.any() or mask.all():
        return out
    idx = np.stack(np.meshgrid(*[np.arange(e) for e in mask.shape], indexing="ij"), -1).reshape(-1, mask.ndim).astype(np.float64)
    flat = mask.reshape(-1)
    d2 = ((idx[:, None, :] - idx[None, :, :]) ** 2).sum(-1)
    d2[flat[:, None] == flat[None, :]] = np.inf
    return np.sqrt(d2.min(1)).astype(np.float32).reshape(mask.shape)


def distance_fields(img: torch.Tensor) -> torch.Tensor:
    """[N, C, ...] -> the fp32 field of ``img > 0.5`` per (n, c), as a tensor of img's device"""
    m = (img.detach() > 0.5).cpu().numpy()
    out = np.zeros(m.shape, dtype=np.float32)
    for n in range(m.shape[0]):
        for c in range(m.shape[1]):
            out[n, c] = mask_field(m[n, c])
    return torch.from_numpy(out).to(img.device)


def activate(logits: torch.Tensor, sigmoid: bool, softmax: bool) -> torch.Tensor:
    if sigmoid:
        return torch.sigmoid(logits)
    if softmax and logits.shape[1] > 1:
        return torch.softmax(logits, dim=1)
    return logits


def kept(p: torch.Tensor, t: torch.Tensor, include_background: bool):
    if not include_background and p.shape[1] > 1:
        return p[:, 1:], t[:, 1:]
    return p, t


def hausdorff_dt_loss(logits: torch.Tensor, target: torch.Tensor, *, alpha: float = 2.0, include_background: bool = False,
                      sigmoid: bool = False, softmax: bool = False, reduction: str = "mean", batch: bool = False,
                      log: bool = False, to_onehot_y: bool = True) -> torch.Tensor:
    """``to_onehot_y`` is accepted for MONAI's call signature; the target's channel count decides (a [N,1,...] target with C > 1
    is a label map)."""
    del to_onehot_y
    p = activate(logits, sigmoid, softmax)
    t = dice_ce_target(logits, target).to(p.dtype)
    p, t = kept(p, t, include_background)
    w = distance_fields(p).to(p.dtype) ** alpha + distance_fields(t).to(p.dtype) ** alpha
    axes = [0] + list(range(2, p.dim())) if batch else list(range(2, p.dim()))
    f = ((p - t) ** 2 * w).mean(dim=axes)
    loss = f.mean() if reduction == "mean" else f.sum()
    return torch.log(loss + 1) if log else loss
