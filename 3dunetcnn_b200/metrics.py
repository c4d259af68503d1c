"""Boundary-distance scores of segmentations on the device: Hausdorff distance (HD, HD95), average surface distance and
normalised surface Dice, as MONAI computes them (``monai/metrics/hausdorff_distance.py``, ``surface_distance.py``,
``surface_dice.py`` and ``utils.py`` of MONAI 1.3+: ``get_mask_edges``, ``get_surface_distance``, ``prepare_spacing``,
``ignore_background``, ``do_metric_reduction``).  Same names, defaults and argument meanings.

MONAI copies each (item, class) pair's masks to the host and runs ``scipy.ndimage.binary_erosion`` and
``distance_transform_edt`` there.  Here one call of libb200unet scores the whole batch: the edges of every pair, an exact
Euclidean distance transform on the device and the reductions, in a fixed number of launches whatever B x C is.  It reads
nothing back to the host: the result is a CUDA tensor, and the call does not synchronise.

Restated semantics:
  * a voxel is foreground iff its value is 1 (MONAI's ``label_idx=1`` after the cast to float): bool True, uint8 1, fp32 1.0;
  * edges = fg & ~erode(fg), 6-neighbour cross, outside the volume = background; distances from each edge voxel of one mask to
    the nearest edge voxel of the other, ``sqrt(((dd s_d)^2 + (dh s_h)^2) + (dw s_w)^2)`` in fp64 rounded to fp32, as scipy
    computes it -- bit for bit with unit spacing;
  * ``percentile`` None or 0 takes the max (MONAI tests ``if not percentile``); otherwise ``torch.quantile`` on the fp32
    distances (rank ``float32(q) * (n - 1)`` in fp32, torch's lerp);
  * both masks empty: nan; exactly one empty: HD and ASD inf, NSD 0.  (With a percentile MONAI takes ``torch.quantile`` of its
    array of infs, whose lerp gives nan; inf is the value that array stands for, and the one returned here.)
  * ASD is the mean over the concatenated distances of the requested directions, in fp64 rounded to fp32.

Limits: 3-D images only (other spatial ranks raise NotImplementedError), 1..256 voxels per axis and at most 4096 (item, class)
pairs per call (RuntimeError from the library beyond them).  Euclidean distances only; ``use_subvoxels`` is not implemented.
Lists of [C, D, H, W] tensors are stacked into one batch (one copy).  No CPU fallback.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np
import torch

from . import lib as _lib
from .prepost import _need_cuda, _plain

__all__ = ["compute_hausdorff_distance", "compute_average_surface_distance", "compute_surface_dice", "prepare_spacing",
           "compute_surface_metrics", "do_metric_reduction", "HausdorffDistanceMetric", "SurfaceDistanceMetric", "SurfaceDiceMetric"]

_REDUCTIONS = ("none", "mean", "sum", "mean_batch", "sum_batch", "mean_channel", "sum_channel")


def prepare_spacing(spacing, batch_size: int, img_dim: int) -> list:
    """MONAI ``prepare_spacing``: None or a number -> the same for every item; ``img_dim`` numbers -> every item;
    ``batch_size`` sequences of ``img_dim`` numbers -> one per item.  Anything else raises ValueError."""
    if spacing is None or isinstance(spacing, (int, float)):
        return [spacing] * batch_size
    if isinstance(spacing, (Sequence, np.ndarray)):
        if len(spacing) == 0:
            raise ValueError("`spacing` must not be empty")
        if any(not isinstance(s, type(spacing[0])) for s in list(spacing)):
            raise ValueError(f"if `spacing` is a sequence, its elements should be of the same type, got {spacing}.")
        if isinstance(spacing[0], (Sequence, np.ndarray)):
            if len(spacing) != batch_size:
                raise ValueError("if `spacing` is a sequence of sequences, the outer sequence should have same length as batch "
                                 f"size ({batch_size}), got {spacing}.")
            if any(len(s) != img_dim for s in list(spacing)):
                raise ValueError(f"each element of `spacing` list should either have same length as image dim ({img_dim}), "
                                 f"got {spacing}.")
            if not all(isinstance(i, (int, float)) for s in list(spacing) for i in list(s)):
                raise ValueError(f"if `spacing` is a sequence of sequences, the inner sequence should contain only int or float "
                                 f"types, got {spacing}.")
            return list(spacing)
        if isinstance(spacing[0], (int, float)):
            if len(spacing) != img_dim:
                raise ValueError(f"if `spacing` is a sequence of numbers, it should have same length as image dim ({img_dim}), "
                                 f"got {spacing}.")
            return [spacing] * batch_size
    raise ValueError(f"`spacing` is a sequence of elements with unsupported type: {type(spacing[0] if len(spacing) else spacing)}")


def _spacing_rows(spacing, batch_size: int) -> np.ndarray:
    rows = []
    for s in prepare_spacing(spacing, batch_size, 3):
        if s is None:
            rows.append((1.0, 1.0, 1.0))
        elif isinstance(s, (int, float)):
            rows.append((float(s),) * 3)
        else:
            rows.append(tuple(float(x) for x in s))
    return np.asarray(rows, dtype=np.float64).reshape(batch_size, 3)


def _as_batch(x, name: str) -> torch.Tensor:
    if isinstance(x, (list, tuple)):
        if not x:
            raise ValueError("%s: empty list" % name)
        return torch.stack([_plain(t) for t in x])
    if not isinstance(x, torch.Tensor):
        raise TypeError("%s: a torch.Tensor or a list of them, got %s" % (name, type(x).__name__))
    return _plain(x)


def _quantile(percentile) -> float:
    if not percentile:
        return 0.0
    if not 0 <= percentile <= 100:
        raise ValueError(f"percentile should be a value between 0 and 100, get {percentile}.")
    return float(np.float32(percentile / 100))


def _check_metric(distance_metric: str) -> None:
    if distance_metric in ("chessboard", "taxicab"):
        raise NotImplementedError("distance_metric=%r: only 'euclidean' distances are implemented" % distance_metric)
    if distance_metric != "euclidean":
        raise ValueError(f"distance_metric {distance_metric} is not implemented.")


def _surface(y_pred, y, include_background: bool, distance_metric: str, spacing, *, q: float = 0.0, hd_dirs: int = 0,
             asd_dirs: int = 0, class_thresholds=None):
    _check_metric(distance_metric)
    y_pred, y = _as_batch(y_pred, "y_pred"), _as_batch(y, "y")
    if y_pred.dim() < 3:
        raise ValueError("y_pred should have at least three dimensions.")
    if y.shape != y_pred.shape:
        raise ValueError(f"y_pred and y should have same shapes, got {y_pred.shape} and {y.shape}.")
    if y_pred.dim() != 5:
        raise NotImplementedError("surface distances are implemented for 3-D images [B, C, D, H, W] only (got %d spatial dims)"
                                  % (y_pred.dim() - 2))
    for name, t in (("y_pred", y_pred), ("y", y)):
        if t.dtype not in _lib._SURFACE_DTYPES:
            raise TypeError("%s: dtype %s; bool, uint8 or float32 masks are supported" % (name, t.dtype))
    if not include_background:
        y = y[:, 1:] if y.shape[1] > 1 else y
        y_pred = y_pred[:, 1:] if y_pred.shape[1] > 1 else y_pred
    b, c = y_pred.shape[:2]
    dev = y_pred.device
    tau = None
    if class_thresholds is not None:
        if len(class_thresholds) != c:
            raise ValueError(f"number of classes ({c}) does not match number of class thresholds ({len(class_thresholds)}).")
        if any(not np.isfinite(t) or t < 0 for t in class_thresholds):
            raise ValueError(f"All class thresholds need to be >= 0 and finite, got {class_thresholds}.")
        tau = torch.tensor([float(t) for t in class_thresholds], dtype=torch.float32)
    rows_np = _spacing_rows(spacing, b)
    if not np.all(np.isfinite(rows_np)):
        raise ValueError(f"spacing must be finite, got {spacing}")
    _need_cuda(y_pred, "surface distance metrics")
    _need_cuda(y, "surface distance metrics")
    if y_pred.device != y.device:
        raise ValueError("y_pred and y are on different devices (%s, %s)" % (y_pred.device, y.device))
    if tau is not None:
        tau = tau.to(dev, non_blocking=True)
    rows = torch.from_numpy(rows_np).to(dev, non_blocking=True)
    out = {k: torch.empty((b, c), dtype=torch.float32, device=dev) if on else None
           for k, on in (("hd", hd_dirs > 0), ("asd", asd_dirs > 0), ("nsd", tau is not None))}
    scratch = torch.empty(_lib.surface_scratch_bytes(b, c, *y_pred.shape[2:]), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.surface_distance(y_pred, y, rows, q, max(hd_dirs, 1), max(asd_dirs, 1), tau, out["hd"], out["asd"], out["nsd"], scratch)
    return out


def compute_hausdorff_distance(y_pred, y, include_background: bool = False, distance_metric: str = "euclidean",
                               percentile: Optional[float] = None, directed: bool = False, spacing=None) -> torch.Tensor:
    """MONAI ``compute_hausdorff_distance``: fp32 [B, C'] on the input's device.  ``directed`` keeps pred -> gt only."""
    q = _quantile(percentile)
    return _surface(y_pred, y, include_background, distance_metric, spacing, q=q, hd_dirs=1 if directed else 2)["hd"]


def compute_average_surface_distance(y_pred, y, include_background: bool = False, symmetric: bool = False,
                                     distance_metric: str = "euclidean", spacing=None) -> torch.Tensor:
    """MONAI ``compute_average_surface_distance``: fp32 [B, C'].  ``symmetric`` averages both directions' distances together."""
    return _surface(y_pred, y, include_background, distance_metric, spacing, asd_dirs=2 if symmetric else 1)["asd"]


def compute_surface_dice(y_pred, y, class_thresholds: Sequence[float], include_background: bool = False,
                         distance_metric: str = "euclidean", spacing=None, use_subvoxels: bool = False) -> torch.Tensor:
    """MONAI ``compute_surface_dice`` (normalised surface Dice, Nikolov et al. 2021): fp32 [B, C'].  ``class_thresholds``: one
    tolerance per scored class (C' entries), compared as float32."""
    if use_subvoxels:
        raise NotImplementedError("use_subvoxels=True (surface areas per edge voxel) is not implemented")
    return _surface(y_pred, y, include_background, distance_metric, spacing, class_thresholds=class_thresholds)["nsd"]


def compute_surface_metrics(y_pred, y, include_background: bool = False, percentile: Optional[float] = None, directed: bool = False,
                            symmetric: bool = False, class_thresholds: Optional[Sequence[float]] = None, spacing=None) -> dict:
    """HD, ASD and (with ``class_thresholds``) NSD from ONE distance transform: {"hd", "asd", "nsd"} -> fp32 [B, C'] each, with
    the arguments of the three functions above."""
    out = _surface(y_pred, y, include_background, "euclidean", spacing, q=_quantile(percentile), hd_dirs=1 if directed else 2,
                   asd_dirs=2 if symmetric else 1, class_thresholds=class_thresholds)
    return {k: v for k, v in out.items() if v is not None}


def do_metric_reduction(f: torch.Tensor, reduction: str = "mean"):
    """MONAI ``do_metric_reduction`` on a [B, C] buffer: nans are left out and counted through ``not_nans``; ``mean`` averages
    over channels first, then over the batch; inf propagates.  Returns (f, not_nans)."""
    reduction = str(getattr(reduction, "value", reduction))
    if reduction not in _REDUCTIONS:
        raise ValueError(f"Unsupported reduction: {reduction}, available options are {list(_REDUCTIONS)}.")
    nans = torch.isnan(f)
    not_nans = ~nans
    t_zero = torch.zeros(1, device=f.device, dtype=torch.float)
    if reduction == "none":
        return f, not_nans.float()
    f = f.clone()
    f[nans] = 0
    if reduction == "mean":
        not_nans = not_nans.sum(dim=1).float()
        f = torch.where(not_nans > 0, f.sum(dim=1).float() / not_nans, t_zero)
        not_nans = (not_nans > 0).sum(dim=0).float()
        f = torch.where(not_nans > 0, f.sum(dim=0).float() / not_nans, t_zero)
    elif reduction == "sum":
        not_nans = not_nans.sum(dim=[0, 1]).float()
        f = torch.sum(f, dim=[0, 1])
    elif reduction == "mean_batch":
        not_nans = not_nans.sum(dim=0).float()
        f = torch.where(not_nans > 0, f.sum(dim=0).float() / not_nans, t_zero)
    elif reduction == "sum_batch":
        not_nans = not_nans.sum(dim=0).float()
        f = f.sum(dim=0).float()
    elif reduction == "mean_channel":
        not_nans = not_nans.sum(dim=1).float()
        f = torch.where(not_nans > 0, f.sum(dim=1).float() / not_nans, t_zero)
    else:   # sum_channel
        not_nans = not_nans.sum(dim=1).float()
        f = f.sum(dim=1).float()
    return f, not_nans


class _CumulativeSurfaceMetric:
    """MONAI's CumulativeIterationMetric surface: ``__call__`` scores a batch and buffers it, ``aggregate`` reduces the buffer."""

    def __init__(self, reduction: str = "mean", get_not_nans: bool = False):
        self.reduction = reduction
        self.get_not_nans = get_not_nans
        self._buffer: list = []

    def _compute(self, y_pred, y, spacing) -> torch.Tensor:
        raise NotImplementedError

    def __call__(self, y_pred, y, spacing=None) -> torch.Tensor:
        r = self._compute(y_pred, y, spacing)
        self._buffer.append(r)
        return r

    def reset(self) -> None:
        self._buffer = []

    def get_buffer(self) -> Optional[torch.Tensor]:
        return torch.cat(self._buffer, dim=0) if self._buffer else None

    def aggregate(self, reduction: Optional[str] = None):
        data = self.get_buffer()
        if not isinstance(data, torch.Tensor):
            raise ValueError("the data to aggregate must be PyTorch Tensor.")
        f, not_nans = do_metric_reduction(data, reduction or self.reduction)
        return (f, not_nans) if self.get_not_nans else f


class HausdorffDistanceMetric(_CumulativeSurfaceMetric):
    """MONAI ``HausdorffDistanceMetric`` on the device."""

    def __init__(self, include_background: bool = False, distance_metric: str = "euclidean", percentile: Optional[float] = None,
                 directed: bool = False, reduction: str = "mean", get_not_nans: bool = False):
        super().__init__(reduction, get_not_nans)
        _check_metric(distance_metric)
        _quantile(percentile)
        self.include_background, self.distance_metric = include_background, distance_metric
        self.percentile, self.directed = percentile, directed

    def _compute(self, y_pred, y, spacing):
        return compute_hausdorff_distance(y_pred, y, self.include_background, self.distance_metric, self.percentile, self.directed,
                                          spacing)


class SurfaceDistanceMetric(_CumulativeSurfaceMetric):
    """MONAI ``SurfaceDistanceMetric`` (average surface distance) on the device."""

    def __init__(self, include_background: bool = False, symmetric: bool = False, distance_metric: str = "euclidean",
                 reduction: str = "mean", get_not_nans: bool = False):
        super().__init__(reduction, get_not_nans)
        _check_metric(distance_metric)
        self.include_background, self.symmetric, self.distance_metric = include_background, symmetric, distance_metric

    def _compute(self, y_pred, y, spacing):
        return compute_average_surface_distance(y_pred, y, self.include_background, self.symmetric, self.distance_metric, spacing)


class SurfaceDiceMetric(_CumulativeSurfaceMetric):
    """MONAI ``SurfaceDiceMetric`` (normalised surface Dice) on the device."""

    def __init__(self, class_thresholds: Sequence[float], include_background: bool = False, distance_metric: str = "euclidean",
                 reduction: str = "mean", get_not_nans: bool = False, use_subvoxels: bool = False):
        super().__init__(reduction, get_not_nans)
        _check_metric(distance_metric)
        if use_subvoxels:
            raise NotImplementedError("use_subvoxels=True (surface areas per edge voxel) is not implemented")
        self.class_thresholds, self.include_background, self.distance_metric = class_thresholds, include_background, distance_metric

    def _compute(self, y_pred, y, spacing):
        return compute_surface_dice(y_pred, y, self.class_thresholds, self.include_background, self.distance_metric, spacing)
