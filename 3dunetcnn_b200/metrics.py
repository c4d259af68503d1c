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

Overlap scores, as MONAI computes them (``monai/metrics/meandice.py``, ``meaniou.py`` and ``confusion_matrix.py`` of MONAI 1.3+):
``DiceHelper`` / ``compute_dice`` / ``DiceMetric``, ``compute_iou`` / ``MeanIoU`` and ``get_confusion_matrix`` /
``compute_confusion_matrix_metric`` / ``ConfusionMatrixMetric``.  One call of libb200unet counts, for every (item, class) pair,
P (predicted voxels), G (target voxels) and I (both) in one pass over the inputs, straight from one-hot masks, label maps or
fp32 logits: no activated, thresholded or one-hot copy of the batch is made.  Each score is a few torch ops on those [B, C]
counts on the device; nothing is read back to the host.

Restated semantics:
  * ``sigmoid=True`` thresholds ``sigmoid(x) > 0.5`` as the compare ``x >= SIGMOID_ABOVE_HALF``, the smallest fp32 whose
    torch.sigmoid on the device is above 0.5 (``x > 0`` differs: the sigmoid of a tiny positive x rounds to 0.5); without
    ``activate`` the values themselves are compared, ``x > 0.5``.  ``softmax=True`` takes the argmax (ties: the lowest channel, as torch.argmax);
  * a label outside [0, C) belongs to no class, in either operand; ``include_background=False`` drops channel 0 after counting.
Deliberate differences from MONAI:
  * a one-hot operand counts its nonzero voxels, so a soft fp32 target is read as binary, where MONAI sums its values (and a
    one-channel input counts nonzero voxels where MONAI compares with 1); ConfusionMatrixMetric does not warn about
    non-binary inputs;
  * the counts are exact integers, where MONAI's fp32 sums stop being exact above 2^24 voxels per pair.
Limits: 3-D images only; 1..128 classes and at most 65535 items per call; label maps uint8 or int64, logits fp32, one-hot masks
bool, uint8 or fp32.  ``GeneralizedDiceScore`` is not provided.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np
import torch

from . import lib as _lib
from .prepost import _need_cuda, _plain

__all__ = ["compute_hausdorff_distance", "compute_average_surface_distance", "compute_surface_dice", "prepare_spacing",
           "compute_surface_metrics", "do_metric_reduction", "HausdorffDistanceMetric", "SurfaceDistanceMetric", "SurfaceDiceMetric",
           "SIGMOID_ABOVE_HALF", "DiceHelper", "compute_dice", "DiceMetric", "compute_iou", "MeanIoU", "get_confusion_matrix",
           "check_confusion_matrix_metric_name", "compute_confusion_matrix_metric", "ConfusionMatrixMetric"]

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


# ---------------------------------------------------------------------------------------------------------- overlap scores
# The smallest fp32 x whose torch.sigmoid(x) on a CUDA tensor is above 0.5 (8.262958e-08).  Below it the device's expf(-x) returns
# 1.0, 1 + exp(-x) is 2 and the sigmoid exactly 0.5.  torch's CPU sigmoid crosses 0.5 higher, at 0x33C00001 (8.940697e-08): its exp
# returns 1 - 2^-24 in between, and 1 + (1 - 2^-24) rounds to 2.  The metrics run on CUDA tensors, so the device's value is taken.
SIGMOID_ABOVE_HALF = float(np.uint32(0x33B17218).view(np.float32))
_ABOVE_HALF = float(np.nextafter(np.float32(0.5), np.float32(1.0)))     # x > 0.5 on values that are already probabilities
_ONEHOT_DTYPES = (torch.bool, torch.uint8, torch.float32)
_LABEL_DTYPES = (torch.bool, torch.uint8, torch.int64)


def _overlap_counts(y_pred, y, n: int, pred_kind: str, threshold: float = 0.0):
    """(P, G, I), int64 [B, n] each, from one pass.  y_pred is read as ``pred_kind``; y [B, 1] with n > 1 is a label map, else
    a one-hot [B, n]."""
    y_pred, y = _as_batch(y_pred, "y_pred"), _as_batch(y, "y")
    if y_pred.dim() < 3:
        raise ValueError(f"y_pred should have at least 3 dimensions (batch, channel, spatial), got {y_pred.dim()}.")
    if y_pred.dim() != 5 or y.dim() != 5:
        raise NotImplementedError("overlap metrics are implemented for 3-D images [B, C, D, H, W] only (got %d and %d spatial dims)"
                                  % (y_pred.dim() - 2, y.dim() - 2))
    if y_pred.shape[0] != y.shape[0] or y_pred.shape[2:] != y.shape[2:]:
        raise ValueError(f"y_pred and y should have the same batch and spatial shape, got {tuple(y_pred.shape)} and {tuple(y.shape)}.")
    gt_kind = "label" if y.shape[1] == 1 and n > 1 else "onehot"
    if not 1 <= n <= 128:
        raise ValueError("%d classes; 1..128 are supported" % n)
    for name, t, kind in (("y_pred", y_pred, pred_kind), ("y", y, gt_kind)):
        want = 1 if kind == "label" else n
        if t.shape[1] != want:
            raise ValueError("%s: %d channels; %s input of %d classes has %d" % (name, t.shape[1], kind, n, want))
        dtypes = {"onehot": _ONEHOT_DTYPES, "label": _LABEL_DTYPES}.get(kind, (torch.float32,))
        if t.dtype not in dtypes:
            raise TypeError("%s: dtype %s; a %s input is %s" % (name, t.dtype, kind, " or ".join(str(d) for d in dtypes)))
    _need_cuda(y_pred, "overlap metrics")
    _need_cuda(y, "overlap metrics")
    if y_pred.device != y.device:
        raise ValueError("y_pred and y are on different devices (%s, %s)" % (y_pred.device, y.device))
    counts = torch.empty((y_pred.shape[0], n, 3), dtype=torch.int64, device=y_pred.device)
    with torch.cuda.device(y_pred.device):
        _lib.overlap_counts(y_pred.contiguous(), pred_kind, y.contiguous(), gt_kind, n, counts, threshold)
    return counts.unbind(-1)


def _overlap_score(num: torch.Tensor, den: torch.Tensor, G: torch.Tensor, P: torch.Tensor, ignore_empty: bool) -> torch.Tensor:
    """num / den in fp32 where the target is not empty; otherwise nan (ignore_empty), 1 when both masks are empty, else 0"""
    if ignore_empty:
        empty = torch.full_like(num, float("nan"), dtype=torch.float32)
    else:
        empty = ((G + P) == 0).float()
    return torch.where(G > 0, num.float() / den.float(), empty)


def _drop_background(counts, include_background: bool):
    return counts if include_background or counts[0].shape[1] == 1 else tuple(t[:, 1:] for t in counts)


class DiceHelper:
    """MONAI ``DiceHelper``: which input form each flag selects, then the Dice of every (item, class) pair and the reduction.
    ``sigmoid`` thresholds at 0.5 (applying the sigmoid only with ``activate``), ``softmax`` takes the argmax over the channels; a
    one-channel ``y_pred`` with ``num_classes > 1`` is a label map.  Returns (f, not_nans) with ``get_not_nans``."""

    def __init__(self, include_background: Optional[bool] = None, sigmoid: bool = False, softmax: Optional[bool] = None,
                 activate: bool = False, get_not_nans: bool = True, reduction: str = "mean_batch", ignore_empty: bool = True,
                 num_classes: Optional[int] = None):
        self.sigmoid = sigmoid
        self.reduction = reduction
        self.get_not_nans = get_not_nans
        self.include_background = sigmoid if include_background is None else include_background
        self.softmax = not sigmoid if softmax is None else softmax
        self.activate = activate
        self.ignore_empty = ignore_empty
        self.num_classes = num_classes

    def counts(self, y_pred, y):
        """(P, G, I) int64 [B, C'] of the classes scored"""
        y_pred = _as_batch(y_pred, "y_pred")
        if y_pred.dim() < 3:
            raise ValueError(f"y_pred should have at least 3 dimensions (batch, channel, spatial), got {y_pred.dim()}.")
        argmax, threshold = self.softmax, self.sigmoid
        n = y_pred.shape[1] if self.num_classes is None else self.num_classes
        if self.num_classes is not None and y_pred.shape[1] == 1 and n > 1:
            argmax = threshold = False
        kind, thr = ("label" if y_pred.shape[1] == 1 and n > 1 else "onehot"), 0.0
        if argmax and n > 1:
            kind = "argmax"
        elif threshold and y_pred.dtype == torch.float32:
            kind, thr = "threshold", SIGMOID_ABOVE_HALF if self.activate else _ABOVE_HALF
        # a bool / uint8 y_pred is above 0.5, or has a sigmoid above 0.5, exactly where it is nonzero: the one-hot reading
        return _drop_background(_overlap_counts(y_pred, y, n, kind, thr), self.include_background)

    def __call__(self, y_pred, y):
        P, G, I = self.counts(y_pred, y)
        f, not_nans = do_metric_reduction(_overlap_score(2 * I, G + P, G, P, self.ignore_empty), self.reduction)
        return (f, not_nans) if self.get_not_nans else f


def compute_dice(y_pred, y, include_background: bool = True, ignore_empty: bool = True, num_classes: Optional[int] = None):
    """MONAI ``compute_dice``: fp32 [B, C'].  ``y_pred`` one-hot [B, C] (nonzero = class) or a label map [B, 1] with
    ``num_classes``; ``y`` one-hot or a label map."""
    return DiceHelper(include_background=include_background, reduction="none", get_not_nans=False, softmax=False,
                      ignore_empty=ignore_empty, num_classes=num_classes)(y_pred, y)


class _CumulativeOverlapMetric(_CumulativeSurfaceMetric):
    """The cumulative base without the surface metrics' spacing argument"""

    def __call__(self, y_pred, y):
        return super().__call__(y_pred, y)


class DiceMetric(_CumulativeOverlapMetric):
    """MONAI ``DiceMetric`` on the device.  ``return_with_label``: True or a list of names turns the aggregate into a dict of
    rounded floats per class (read back to the host, as MONAI does)."""

    def __init__(self, include_background: bool = True, reduction: str = "mean", get_not_nans: bool = False, ignore_empty: bool = True,
                 num_classes: Optional[int] = None, return_with_label=False):
        super().__init__(reduction, get_not_nans)
        self.include_background, self.ignore_empty, self.num_classes = include_background, ignore_empty, num_classes
        self.return_with_label = return_with_label

    def _compute(self, y_pred, y, spacing):
        return compute_dice(y_pred, y, self.include_background, self.ignore_empty, self.num_classes)

    def aggregate(self, reduction: Optional[str] = None):
        data = self.get_buffer()
        if not isinstance(data, torch.Tensor):
            raise ValueError("the data to aggregate must be PyTorch Tensor.")
        f, not_nans = do_metric_reduction(data, reduction or self.reduction)
        if self.return_with_label:
            if isinstance(self.return_with_label, bool):
                first = 0 if self.include_background else 1
                f = {f"label_{i + first}": round(v.item(), 4) for i, v in enumerate(f)}
            else:
                f = {key: round(v.item(), 4) for key, v in zip(self.return_with_label, f)}
        return (f, not_nans) if self.get_not_nans else f


def _same_shape_counts(y_pred, y, include_background: bool):
    y_pred, y = _as_batch(y_pred, "y_pred"), _as_batch(y, "y")
    if y.shape != y_pred.shape:
        raise ValueError(f"y_pred and y should have same shapes, got {y_pred.shape} and {y.shape}.")
    if y_pred.dim() < 3:
        raise ValueError(f"y_pred should have at least 3 dimensions (batch, channel, spatial), got {y_pred.dim()}.")
    return _drop_background(_overlap_counts(y_pred, y, y_pred.shape[1], "onehot"), include_background), y_pred.shape[2:].numel()


def compute_iou(y_pred, y, include_background: bool = True, ignore_empty: bool = True) -> torch.Tensor:
    """MONAI ``compute_iou``: fp32 [B, C'] of one-hot inputs of the same shape (nonzero = class)."""
    (P, G, I), _ = _same_shape_counts(y_pred, y, include_background)
    return _overlap_score(I, G + P - I, G, P, ignore_empty)


class MeanIoU(_CumulativeOverlapMetric):
    """MONAI ``MeanIoU`` on the device."""

    def __init__(self, include_background: bool = True, reduction: str = "mean", get_not_nans: bool = False, ignore_empty: bool = True):
        super().__init__(reduction, get_not_nans)
        self.include_background, self.ignore_empty = include_background, ignore_empty

    def _compute(self, y_pred, y, spacing):
        return compute_iou(y_pred, y, self.include_background, self.ignore_empty)


def get_confusion_matrix(y_pred, y, include_background: bool = True) -> torch.Tensor:
    """MONAI ``get_confusion_matrix``: fp32 [B, C', 4] = (tp, fp, tn, fn) of one-hot inputs of the same shape, each the exact
    count rounded once to fp32."""
    (P, G, I), S = _same_shape_counts(y_pred, y, include_background)
    return torch.stack([I, P - I, S - P - G + I, G - I], dim=-1).float()


_CM_NAMES = {
    "tpr": ("sensitivity", "recall", "hit_rate", "true_positive_rate", "tpr"),
    "tnr": ("specificity", "selectivity", "true_negative_rate", "tnr"),
    "ppv": ("precision", "positive_predictive_value", "ppv"),
    "npv": ("negative_predictive_value", "npv"),
    "fnr": ("miss_rate", "false_negative_rate", "fnr"),
    "fpr": ("fall_out", "false_positive_rate", "fpr"),
    "fdr": ("false_discovery_rate", "fdr"),
    "for": ("false_omission_rate", "for"),
    "pt": ("prevalence_threshold", "pt"),
    "ts": ("threat_score", "critical_success_index", "ts", "csi"),
    "acc": ("accuracy", "acc"),
    "ba": ("balanced_accuracy", "ba"),
    "f1": ("f1_score", "f1"),
    "mcc": ("matthews_correlation_coefficient", "mcc"),
    "fm": ("fowlkes_mallows_index", "fm"),
    "bm": ("informedness", "bookmaker_informedness", "bm", "youden_index", "youden"),
    "mk": ("markedness", "deltap", "mk"),
}


def check_confusion_matrix_metric_name(metric_name: str) -> str:
    """MONAI's names and aliases -> the short name; spaces count as underscores, case is ignored"""
    name = metric_name.replace(" ", "_").lower()
    for short, aliases in _CM_NAMES.items():
        if name in aliases:
            return short
    raise NotImplementedError("the metric is not implemented.")


def compute_confusion_matrix_metric(metric_name: str, confusion_matrix: torch.Tensor) -> torch.Tensor:
    """MONAI ``compute_confusion_matrix_metric`` on [..., 4] (tp, fp, tn, fn): nan where a denominator is 0."""
    metric = check_confusion_matrix_metric_name(metric_name)
    if confusion_matrix.dim() == 1:
        confusion_matrix = confusion_matrix.unsqueeze(dim=0)
    if confusion_matrix.shape[-1] != 4:
        raise ValueError("the size of the last dimension of confusion_matrix should be 4.")
    tp, fp, tn, fn = confusion_matrix.unbind(-1)
    p, n = tp + fn, fp + tn
    nan = torch.tensor(float("nan"), device=confusion_matrix.device)

    def ratio(a, b):
        return torch.where(b > 0, a / b, nan)

    if metric in ("pt", "ba", "bm"):
        tpr, tnr = ratio(tp, p), ratio(tn, n)
        if metric == "pt":
            num, den = torch.sqrt(tpr * (1.0 - tnr)) + tnr - 1.0, tpr + tnr - 1.0
        else:
            return (tpr + tnr) / 2.0 if metric == "ba" else tpr + tnr - 1.0
    elif metric == "fm":
        return torch.sqrt(ratio(tp, tp + fp) * ratio(tp, p))
    elif metric == "mk":
        return ratio(tp, tp + fp) + ratio(tn, tn + fn) - 1.0
    elif metric == "mcc":
        num, den = tp * tn - fp * fn, torch.sqrt((tp + fp) * (tp + fn) * (tn + fp) * (tn + fn))
    else:
        num, den = {"tpr": (tp, p), "tnr": (tn, n), "ppv": (tp, tp + fp), "npv": (tn, tn + fn), "fnr": (fn, p), "fpr": (fp, n),
                    "fdr": (fp, fp + tp), "for": (fn, fn + tn), "ts": (tp, tp + fn + fp), "acc": (tp + tn, p + n),
                    "f1": (tp * 2.0, tp * 2.0 + fn + fp)}[metric]
    return torch.where(den != 0, num / den, nan)


class ConfusionMatrixMetric(_CumulativeOverlapMetric):
    """MONAI ``ConfusionMatrixMetric`` on the device.  The buffer holds [B, C', 4] matrices; ``aggregate`` returns one result per
    name: with ``compute_sample`` the metric of each sample, then the reduction; otherwise the reduction of the matrices, then the
    metric."""

    def __init__(self, include_background: bool = True, metric_name="hit_rate", compute_sample: bool = False, reduction: str = "mean",
                 get_not_nans: bool = False):
        super().__init__(reduction, get_not_nans)
        self.include_background = include_background
        self.metric_name = (metric_name,) if isinstance(metric_name, str) else tuple(metric_name)
        for name in self.metric_name:
            check_confusion_matrix_metric_name(name)
        self.compute_sample = compute_sample

    def _compute(self, y_pred, y, spacing):
        return get_confusion_matrix(y_pred, y, self.include_background)

    def aggregate(self, compute_sample: bool = False, reduction: Optional[str] = None):
        data = self.get_buffer()
        if not isinstance(data, torch.Tensor):
            raise ValueError("the data to aggregate must be PyTorch Tensor.")
        results = []
        for name in self.metric_name:
            if compute_sample or self.compute_sample:
                f, not_nans = do_metric_reduction(compute_confusion_matrix_metric(name, data), reduction or self.reduction)
            else:
                f, not_nans = do_metric_reduction(data, reduction or self.reduction)
                f = compute_confusion_matrix_metric(name, f)
            results.append((f, not_nans) if self.get_not_nans else f)
        return results
