"""Random augmentation of a training batch on the device: the spatial and intensity transforms that
``unet3d/datasets/segmentation.py:72-94`` (paths relative to /root/reference) chains after loading, under MONAI's names
and keyword arguments, fused into two passes over the image (``csrc/augment.cu``).

  * ``RandFlipd`` / ``RandRotated`` (``keys=("image", "label")``): composed per sample into one 3x4 index-space affine
    (output index -> source index), as MONAI's lazy resampling composes them, and applied by one resample: trilinear for
    the fp32 image, nearest for the uint8 label.  Output shape = input shape (``keep_size=True``).
  * ``NormalizeIntensityd`` (z-score), then ``RandScaleIntensityd`` / ``RandShiftIntensityd`` (``keys=("image",)``): the
    resample pass also sums the statistics of the resampled image; a second pass applies ``((x - mean) / std) * a + b``
    in place, (a, b) per (sample, channel) holding the composed scale / shift.

Decisions (MONAI is not installed here, so parity with it is unpinned; the semantics are restated from its public source):
  * Labels are resampled nearest and stay uint8, so they remain targets of the fused Dice kernels.  The label key of
    ``RandRotated`` accepts ``mode`` omitted or ``"nearest"`` (e.g. ``mode=("bilinear", "nearest")``); anything else raises
    ``NotImplementedError``.  Images are resampled trilinear (``"bilinear"``, MONAI's name for it in 3D).
  * ``keep_size=False``, ``align_corners=True``, ``padding_mode="reflection"``, non-fp32 images, non-uint8 labels and
    transform names other than the five above raise.
  * Random parameters come from one CPU ``torch.Generator`` per ``Compose``: per sample, per transform in order, first the
    ``prob`` draw, then (when the transform fires) its values.  ``set_random_state(seed)`` makes a run reproducible; give
    each data-parallel rank its own seed.  The sequences are not MONAI's numpy streams.
  * Each call uploads the drawn affines and intensity coefficients in one non-blocking copy from pinned memory and never
    synchronises the host.  The draws of the last call stay readable as ``last_params``.

Geometry stage (``csrc/foreground.cu``): ``CropForegroundd`` then ``Resized``, the crop and resize of
``segmentation.py:55-70``, ahead of the spatial transforms.  MONAI composes them lazily with the flips and the rotation, so
the batch is interpolated once; so does this stage:
  * Threshold (the reference's ``utils/threshold.py:6-15`` ``percentile_threshold(p)``): per (sample, channel)
    ``thr = np.percentile(x.flatten(), p * 100)``, method "linear", bit for bit.  numpy (2.x) divides ``p * 100`` by the
    data's ``dtype.type(100)``, so for fp32 images the virtual index ``(n - 1) * q``, its weight and the interpolation
    ``_lerp`` all run in fp32 (``percentile_index`` restates the index arithmetic; the device finds the two order statistics
    by an exact radix select).  A NaN in a channel makes its ``thr`` NaN: it selects nothing.  ``foreground_percentile=None``
    is MONAI's default ``select_fn`` (``x > 0``).
  * Box (MONAI ``generate_spatial_bounding_box``): mask ``any_c(x_c > thr_c)``; per axis ``[first - margin, last + margin +
    1)``, clipped to the volume when ``allow_smaller`` (otherwise the box may pass the edge and the ``Compose``'s padding
    mode supplies the outside).  Deviation: MONAI returns a zero-size box for an empty mask, which ``Resized`` cannot use;
    here the whole volume is used and the sample is flagged in ``last_params["empty"]`` (raising would need a host sync).
  * One resample: with box start b, size B, output size O, s = B / O and the drawn affine A (index space on the O grid),
    output index p reads source index ``b + s (A p) + (s - 1) / 2`` -- MONAI's lazy ``Resize`` (= ``interpolate(
    align_corners=False)``) after the crop's translation.  Samples read their full volume: voxels just outside the box are
    real data, as under lazy resampling.  The flips and the rotation are drawn on the O grid (rotation centre (O - 1) / 2).
  * The batch may be a list of (C, D_i, H_i, W_i) tensors of different extents (``list_collate``); the output is one batch.
"""
from __future__ import annotations

import copy
import math
from typing import Sequence

import numpy as np
import torch

from . import lib as _lib
from .prepost import _need_cuda, _plain

_PADDING = {"border": 0, "zeros": 1}


def _keys(keys) -> tuple:
    return (keys,) if isinstance(keys, str) else tuple(keys)


def _uniform_range(v, what: str) -> tuple:
    """A scalar r means U(-r, r), a pair U(lo, hi)."""
    if isinstance(v, (int, float)):
        return (min(-float(v), float(v)), max(-float(v), float(v)))
    v = tuple(float(x) for x in v)
    if len(v) == 1:
        return (min(-v[0], v[0]), max(-v[0], v[0]))
    if len(v) != 2:
        raise ValueError("%s: a scalar or a (low, high) pair, got %r" % (what, v))
    return (min(v), max(v))


def _rand(g: torch.Generator) -> float:
    return float(torch.rand((), generator=g, dtype=torch.float64))


def _uniform(g: torch.Generator, lo_hi) -> float:
    return lo_hi[0] + (lo_hi[1] - lo_hi[0]) * _rand(g)


class _Transform:
    """A transform is a parameter sampler; running it alone runs a one-element ``Compose``."""
    kind = None     # "spatial", "normalize" or "intensity"
    _own = None

    def __call__(self, data):
        if self._own is None:
            self._own = Compose([self])
        return self._own(data)

    def set_random_state(self, seed=None):
        if self._own is None:
            self._own = Compose([self])
        self._own.set_random_state(seed)
        return self


class RandFlipd(_Transform):
    """``monai.transforms.RandFlipd``: with probability ``prob`` flip the listed spatial axes (0 = D); ``None`` flips all three."""
    kind = "spatial"

    def __init__(self, keys, prob: float = 0.1, spatial_axis=None, allow_missing_keys: bool = False, lazy: bool = False):
        self.keys, self.prob = _keys(keys), float(prob)
        axes = (0, 1, 2) if spatial_axis is None else ((spatial_axis,) if isinstance(spatial_axis, int) else tuple(spatial_axis))
        if any(a not in (0, 1, 2, -1, -2, -3) for a in axes):
            raise ValueError("RandFlipd: spatial_axis must be in 0..2 (or -3..-1), got %r" % (spatial_axis,))
        self.axes = tuple(sorted({a % 3 for a in axes}))
        self.padding_mode = None

    def draw(self, g: torch.Generator, n_channels: int) -> dict:
        return {"name": "RandFlipd", "do": _rand(g) < self.prob, "axes": self.axes}

    @staticmethod
    def matrix(params: dict, spatial: Sequence[int]) -> np.ndarray:
        m = np.eye(4)
        if params["do"]:
            for a in params["axes"]:
                m[a, a] = -1.0
                m[a, 3] = spatial[a] - 1.0
        return m


def rotation_matrix(angles) -> np.ndarray:
    """MONAI ``create_rotate`` for three angles (radians) in array axis order D, H, W: R = Rx @ Ry @ Rz (3 x 3)."""
    x, y, z = (float(a) for a in angles)
    rx = np.array([[1, 0, 0], [0, math.cos(x), -math.sin(x)], [0, math.sin(x), math.cos(x)]])
    ry = np.array([[math.cos(y), 0, math.sin(y)], [0, 1, 0], [-math.sin(y), 0, math.cos(y)]])
    rz = np.array([[math.cos(z), -math.sin(z), 0], [math.sin(z), math.cos(z), 0], [0, 0, 1]])
    return rx @ ry @ rz


class RandRotated(_Transform):
    """``monai.transforms.RandRotated``: with probability ``prob`` rotate about the volume centre c = (size - 1) / 2 by angles
    drawn from ``range_x``, ``range_y``, ``range_z`` (a scalar r means U(-r, r), a pair U(lo, hi)); the source index of output
    index p is c + R (p - c).  ``padding_mode`` "border" (MONAI's default) or "zeros"."""
    kind = "spatial"

    def __init__(self, keys, range_x=0.0, range_y=0.0, range_z=0.0, prob: float = 0.1, keep_size: bool = True,
                 mode=None, padding_mode="border", align_corners=False, dtype=None, allow_missing_keys: bool = False,
                 lazy: bool = False):
        self.keys, self.prob = _keys(keys), float(prob)
        self.ranges = tuple(_uniform_range(r, "RandRotated range") for r in (range_x, range_y, range_z))
        if not keep_size:
            raise NotImplementedError("RandRotated: keep_size=False is not implemented (the output keeps the input's shape)")
        if any(bool(a) for a in (align_corners if isinstance(align_corners, (list, tuple)) else (align_corners,))):
            raise NotImplementedError("RandRotated: align_corners=True is not implemented")
        modes = _keys(mode) if mode is not None else (None,) * len(self.keys)
        if len(modes) == 1:
            modes = modes * len(self.keys)
        for k, m in zip(self.keys, modes):
            if k == "label" and m not in (None, "nearest"):
                raise NotImplementedError("RandRotated: the label is resampled nearest and stays uint8; mode %r is not "
                                          "implemented for it" % (m,))
            if k != "label" and m not in (None, "bilinear", "trilinear"):
                raise NotImplementedError("RandRotated: the image is resampled trilinear ('bilinear'); mode %r is not "
                                          "implemented" % (m,))
        pads = set(_keys(padding_mode))
        if len(pads) != 1 or not pads <= set(_PADDING):
            raise NotImplementedError("RandRotated: padding_mode 'border' or 'zeros' (one for every key), got %r" % (padding_mode,))
        self.padding_mode = pads.pop()

    def draw(self, g: torch.Generator, n_channels: int) -> dict:
        do = _rand(g) < self.prob
        angles = tuple(_uniform(g, r) for r in self.ranges) if do else (0.0, 0.0, 0.0)
        return {"name": "RandRotated", "do": do, "angles": angles}

    @staticmethod
    def matrix(params: dict, spatial: Sequence[int]) -> np.ndarray:
        m = np.eye(4)
        if params["do"]:
            r = rotation_matrix(params["angles"])
            c = (np.asarray(spatial, dtype=np.float64) - 1.0) / 2.0
            m[:3, :3] = r
            m[:3, 3] = c - r @ c
        return m


class NormalizeIntensityd(_Transform):
    """``monai.transforms.NormalizeIntensityd``: (x - mean) / std (population std, std 0 -> 1) per sample, per channel when
    ``channel_wise``; ``nonzero``: statistics over, and changes to, the non-zero voxels only."""
    kind = "normalize"

    def __init__(self, keys, subtrahend=None, divisor=None, nonzero: bool = False, channel_wise: bool = False, dtype=None,
                 allow_missing_keys: bool = False):
        if subtrahend is not None or divisor is not None:
            raise NotImplementedError("NormalizeIntensityd: explicit subtrahend/divisor are not implemented")
        self.keys, self.nonzero, self.channel_wise = _keys(keys), bool(nonzero), bool(channel_wise)
        self.prob = 1.0


class _RandIntensity(_Transform):
    kind = "intensity"
    _arg = None

    def __init__(self, keys, value, prob: float = 0.1, channel_wise: bool = False, allow_missing_keys: bool = False):
        self.keys, self.prob, self.channel_wise = _keys(keys), float(prob), bool(channel_wise)
        self.range = _uniform_range(value, "%s %s" % (type(self).__name__, self._arg))

    def draw(self, g: torch.Generator, n_channels: int) -> dict:
        do = _rand(g) < self.prob
        vals = [_uniform(g, self.range) for _ in range(n_channels if self.channel_wise else 1)] if do else [0.0]
        if len(vals) == 1:
            vals = vals * n_channels
        return {"name": type(self).__name__, "do": do, self._arg: vals}


class RandScaleIntensityd(_RandIntensity):
    """``monai.transforms.RandScaleIntensityd``: x * (1 + f), f ~ U(-factors, factors) or U(lo, hi), per channel when
    ``channel_wise``."""
    _arg = "factors"

    def __init__(self, keys, factors, prob: float = 0.1, channel_wise: bool = False, dtype=None, allow_missing_keys: bool = False):
        super().__init__(keys, factors, prob, channel_wise, allow_missing_keys)

    @staticmethod
    def update(params: dict, a: np.ndarray, b: np.ndarray) -> None:
        s = 1.0 + np.asarray(params["factors"])
        a *= s
        b *= s


class RandShiftIntensityd(_RandIntensity):
    """``monai.transforms.RandShiftIntensityd``: x + o, o ~ U(-offsets, offsets) or U(lo, hi), per channel when
    ``channel_wise``."""
    _arg = "offsets"

    def __init__(self, keys, offsets, safe: bool = False, prob: float = 0.1, channel_wise: bool = False,
                 allow_missing_keys: bool = False):
        super().__init__(keys, offsets, prob, channel_wise, allow_missing_keys)

    @staticmethod
    def update(params: dict, a: np.ndarray, b: np.ndarray) -> None:
        b += np.asarray(params["offsets"])


def percentile_index(size: int, q: float):
    """The index arithmetic of ``np.percentile(x, q * 100)`` (method "linear") for fp32 data of ``size`` elements, from the
    size alone: ``(lower rank, upper rank, weight)``, weight a ``np.float32``.  The percentile is then
    ``_lerp(sorted[lower], sorted[upper], weight)`` in fp32.  The same operations numpy runs (numpy 2 promotion rules)."""
    qf = np.true_divide(q * 100, np.float32(100), out=...)          # np.percentile: q / dtype.type(100) -> fp32
    vi = (size - 1) * qf                                             # _quantile: linear virtual index, fp32
    if vi >= size - 1:
        prev, lo, hi = -1, size - 1, size - 1                        # _get_indexes: above the last index -> index -1
    elif vi < 0:
        prev, lo, hi = 0, 0, 0
    else:
        prev = int(np.floor(vi))
        lo, hi = prev, prev + 1
    gamma = np.asanyarray(vi - np.asarray(prev, dtype=np.intp), dtype=vi.dtype)   # _get_gamma, cast back to fp32
    return lo, hi, np.float32(gamma)


class CropForegroundd(_Transform):
    """``monai.transforms.CropForegroundd`` with ``select_fn`` the reference's ``percentile_threshold(foreground_percentile)``
    or, for ``None``, MONAI's default ``x > 0``.  The crop is applied by the following ``Resized`` (see the module docstring)."""
    kind = "crop"

    def __init__(self, keys, source_key: str = "image", foreground_percentile=None, margin: int = 1, allow_smaller: bool = True,
                 select_fn=None, k_divisible=1, allow_missing_keys: bool = False, lazy: bool = False):
        self.keys = _keys(keys)
        if source_key != "image":
            raise NotImplementedError("CropForegroundd: source_key must be 'image', got %r" % (source_key,))
        if select_fn is not None:
            raise NotImplementedError("CropForegroundd: arbitrary select_fn callables run on the host; give foreground_percentile "
                                      "(percentile_threshold) or None (x > 0)")
        if any(int(k) != 1 for k in (k_divisible if isinstance(k_divisible, (list, tuple)) else (k_divisible,))):
            raise NotImplementedError("CropForegroundd: k_divisible other than 1 is not implemented")
        if foreground_percentile is not None and not 0.0 <= float(foreground_percentile) <= 1.0:
            raise ValueError("CropForegroundd: foreground_percentile in [0, 1], got %r" % (foreground_percentile,))
        if int(margin) < 0:
            raise ValueError("CropForegroundd: margin >= 0, got %r" % (margin,))
        self.percentile = None if foreground_percentile is None else float(foreground_percentile)
        self.margin, self.allow_smaller = int(margin), bool(allow_smaller)
        self.padding_mode = None


class Resized(_Transform):
    """``monai.transforms.Resized`` to ``spatial_size`` (three positive ints): trilinear for the image, nearest for the label."""
    kind = "resize"

    def __init__(self, keys, spatial_size, mode=("trilinear", "nearest"), size_mode: str = "all", align_corners=None,
                 anti_aliasing: bool = False, dtype=None, allow_missing_keys: bool = False, lazy: bool = False):
        self.keys = _keys(keys)
        size = (int(spatial_size),) * 3 if isinstance(spatial_size, int) else tuple(int(v) for v in spatial_size)
        if len(size) != 3 or min(size) < 1:
            raise NotImplementedError("Resized: spatial_size must be three positive sizes, got %r" % (spatial_size,))
        if size_mode != "all":
            raise NotImplementedError("Resized: size_mode %r is not implemented" % (size_mode,))
        if anti_aliasing:
            raise NotImplementedError("Resized: anti_aliasing is not implemented")
        if any(bool(a) for a in (align_corners if isinstance(align_corners, (list, tuple)) else (align_corners,))):
            raise NotImplementedError("Resized: align_corners=True is not implemented")
        modes = _keys(mode)
        if len(modes) == 1:
            modes = modes * len(self.keys)
        for k, m in zip(self.keys, modes):
            if k == "label" and m != "nearest":
                raise NotImplementedError("Resized: the label is resampled nearest and stays uint8; mode %r is not implemented "
                                          "for it" % (m,))
            if k != "label" and m not in ("bilinear", "trilinear"):
                raise NotImplementedError("Resized: the image is resampled trilinear; mode %r is not implemented" % (m,))
        self.spatial_size = size
        self.padding_mode = None


def list_collate(batch):
    """``DataLoader`` ``collate_fn`` that keeps ``"image"`` and ``"label"`` as lists of per-sample tensors (volumes of different
    sizes cannot be stacked; the device ``Compose`` with a ``Resized`` stacks them) and collates every other entry as the
    default collate does."""
    from torch.utils.data import default_collate
    out = {}
    for k in batch[0]:
        vals = [b[k] for b in batch]
        out[k] = [torch.as_tensor(v) for v in vals] if k in ("image", "label") else default_collate(vals)
    return out


# MONAI exports both spellings; the reference's configs use the "D" one
RandFlipD, RandRotateD, NormalizeIntensityD = RandFlipd, RandRotated, NormalizeIntensityd
RandScaleIntensityD, RandShiftIntensityD = RandScaleIntensityd, RandShiftIntensityd
CropForegroundD, ResizeD = CropForegroundd, Resized
_BY_NAME = {c.__name__: c for c in (RandFlipd, RandRotated, NormalizeIntensityd, RandScaleIntensityd, RandShiftIntensityd)}
_BY_NAME.update({k[:-1] + "D": v for k, v in list(_BY_NAME.items())})
_SPATIAL_KEYS = (("image",), ("image", "label"))


class Compose:
    """The transforms of one batch in two device passes.  Order: spatial transforms (fused into one affine per sample), at
    most one ``NormalizeIntensityd``, then the intensity transforms (fused into one (a, b) per sample and channel) -- the
    order ``segmentation.py:72-94`` builds.  Spatial transforms act on ``("image",)`` or ``("image", "label")``, the others
    on ``("image",)``.

    Call it on a dict with an fp32 CUDA ``"image"`` (N, C, D, H, W) or (C, D, H, W) and, when the spatial keys name it, a
    uint8 ``"label"`` of the same spatial shape (a one-hot target or a one-channel label map).  Returns a new dict with
    plain tensors of the same shapes and dtypes; other entries pass through.

    An optional geometry stage comes first: at most one ``CropForegroundd``, then exactly one ``Resized``.  With it the
    ``"image"`` may also be a list of (C, D_i, H_i, W_i) CUDA tensors of different extents (the ``"label"`` then a list of
    the same form), and the result is one (N, C) + ``spatial_size`` batch.  ``last_params`` then also holds, on the device,
    ``box`` int32 [N][3][2] (start, end), ``empty`` int32 [N], ``threshold`` fp32 [N][C] (with a ``foreground_percentile``)
    and ``source_affine`` fp32 [N][3][4] (output index -> index in the sample's own volume)."""

    def __init__(self, transforms):
        self.transforms = list(transforms)
        stage = {"crop": -2, "resize": -1, "spatial": 0, "normalize": 1, "intensity": 2}
        last = -3
        for t in self.transforms:
            if not isinstance(t, _Transform):
                raise ValueError("Compose: %r is not a device transform of this module" % (t,))
            s = stage[t.kind]
            if s < last or (s == last and t.kind in ("crop", "resize", "normalize")):
                raise ValueError("Compose: the order is at most one CropForegroundd, one Resized, spatial transforms, at most one "
                                 "NormalizeIntensityd, then intensity transforms; got %s" % [type(x).__name__ for x in self.transforms])
            last = s
            if t.kind not in ("spatial", "crop", "resize") and t.keys != ("image",):
                raise ValueError("%s: keys must be ('image',), got %r" % (type(t).__name__, t.keys))
        self.spatial = [t for t in self.transforms if t.kind == "spatial"]
        self.intensity = [t for t in self.transforms if t.kind == "intensity"]
        norms = [t for t in self.transforms if t.kind == "normalize"]
        self.normalize = norms[0] if norms else None
        crops = [t for t in self.transforms if t.kind == "crop"]
        resizes = [t for t in self.transforms if t.kind == "resize"]
        if crops and not resizes:
            raise ValueError("Compose: a CropForegroundd needs a Resized after it (the batch is stacked at its spatial_size)")
        self.crop = crops[0] if crops else None
        self.resize = resizes[0] if resizes else None
        keys = {t.keys for t in self.spatial + crops + resizes}
        if len(keys) > 1 or not keys <= set(_SPATIAL_KEYS):
            raise ValueError("Compose: every crop, resize and spatial transform takes keys ('image',) or ('image', 'label'), all "
                             "the same; got %s" % sorted(keys))
        self.spatial_keys = keys.pop() if keys else ("image",)
        pads = {t.padding_mode for t in self.spatial if t.padding_mode is not None}
        if len(pads) > 1:
            raise ValueError("Compose: the rotations of one Compose share one padding_mode, got %s" % sorted(pads))
        self.padding_mode = pads.pop() if pads else "border"
        self.generator = torch.Generator()
        self.generator.seed()
        self.last_params = None
        self.last_stats = None

    def set_random_state(self, seed=None):
        """Seed the generator of the draws (None: a non-deterministic seed)."""
        if seed is None:
            self.generator.seed()
        else:
            self.generator.manual_seed(int(seed))
        return self

    def draw(self, n: int, n_channels: int, spatial: Sequence[int]) -> dict:
        """The parameters of one batch (host only): per sample, per transform in order.  ``matrices`` [n][spatial][4][4] and
        their product in application order ``affine`` [n][3][4] (fp64, output index -> source index); ``coef`` [n][C][2]
        (a, b) of the composed intensity transforms."""
        per_sample, mats, affine = [], [], []
        coef = np.zeros((n, n_channels, 2))
        for i in range(n):
            rec = []
            a, b = np.ones(n_channels), np.zeros(n_channels)
            ms, m = [], np.eye(4)
            for t in self.transforms:
                if t.kind in ("normalize", "crop", "resize"):
                    rec.append({"name": type(t).__name__, "do": True})
                    continue
                p = t.draw(self.generator, n_channels)
                rec.append(p)
                if t.kind == "spatial":
                    ms.append(t.matrix(p, spatial))
                    m = m @ ms[-1]          # y_k(p) = y_{k-1}(M_k p): later transforms multiply on the right
                elif p["do"]:
                    t.update(p, a, b)
            per_sample.append(rec)
            mats.append(np.stack(ms) if ms else np.zeros((0, 4, 4)))
            affine.append(m[:3])
            coef[i, :, 0], coef[i, :, 1] = a, b
        return {"transforms": per_sample, "matrices": [torch.from_numpy(x) for x in mats],
                "affine": torch.from_numpy(np.stack(affine)), "coef": torch.from_numpy(coef), "padding_mode": self.padding_mode,
                "normalize": None if self.normalize is None else {"nonzero": self.normalize.nonzero,
                                                                   "channel_wise": self.normalize.channel_wise}}

    def __call__(self, data):
        if self.resize is not None:
            return self._call_geometry(data)
        img = _plain(data["image"])
        _need_cuda(img, "augment.Compose")
        if img.dtype != torch.float32:
            raise NotImplementedError("augment: the image must be fp32, got %s" % img.dtype)
        batched = img.dim() == 5
        if img.dim() not in (4, 5):
            raise ValueError("augment: image (N, C, D, H, W) or (C, D, H, W), got shape %s" % (tuple(img.shape),))
        x = (img if batched else img[None]).contiguous()
        n, c, d, h, w = x.shape
        lab = None
        if "label" in self.spatial_keys:
            lab = _plain(data["label"])
            _need_cuda(lab, "augment.Compose")
            if lab.dtype != torch.uint8:
                raise NotImplementedError("augment: the label must be uint8 (one-hot or label map), got %s" % lab.dtype)
            lab = (lab if batched else lab[None]).contiguous()
            if lab.dim() != 5 or lab.shape[0] != n or tuple(lab.shape[2:]) != (d, h, w):
                raise ValueError("augment: label shape %s does not match image shape %s" % (tuple(lab.shape), tuple(x.shape)))
        params = self.draw(n, c, (d, h, w))
        host = torch.empty(n * 12 + n * c * 2, dtype=torch.float32, pin_memory=True)
        host[: n * 12] = params["affine"].reshape(-1)
        host[n * 12:] = params["coef"].reshape(-1)
        dev = host.to(x.device, non_blocking=True)
        out = torch.empty_like(x)
        lout = torch.empty_like(lab) if lab is not None else None
        norm = self.normalize
        with torch.cuda.device(x.device):
            lib = _lib.load_library()
            nbytes = int(lib.b200unet_augment_scratch_bytes(n, c, d * h * w))
            if nbytes == 0:
                raise ValueError("augment: %s" % lib.b200unet_last_error().decode())
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
            _lib.check(lib.b200unet_augment_resample(x.data_ptr(), lab.data_ptr() if lab is not None else None, n, c,
                                                     lab.shape[1] if lab is not None else 0, d, h, w, dev.data_ptr(),
                                                     _PADDING[self.padding_mode], int(norm is not None and norm.nonzero),
                                                     out.data_ptr(), lout.data_ptr() if lout is not None else None,
                                                     scratch.data_ptr(), _lib.stream_ptr()), "augment_resample")
            if norm is not None or self.intensity:
                _lib.check(lib.b200unet_augment_intensity(out.data_ptr(), n, c, d * h * w, int(norm is not None),
                                                          int(norm is not None and norm.nonzero),
                                                          int(norm is not None and norm.channel_wise),
                                                          dev.data_ptr() + 4 * n * 12, scratch.data_ptr(), _lib.stream_ptr()),
                           "augment_intensity")
        self.last_params = params
        self.last_stats = scratch[: 8 * 3 * n * c].view(torch.float64).view(n, c, 3) if norm is not None else None
        res = dict(data)
        res["image"] = out if batched else out[0]
        if lout is not None:
            res["label"] = lout if batched else lout[0]
        return res


    def _samples(self, data):
        """(images, labels or None, batched): per-sample (C, D, H, W) views of a 5-D batch or the tensors of a list"""
        img = data["image"]
        listed = isinstance(img, (list, tuple))
        if listed:
            imgs = [_plain(t) for t in img]
        else:
            img = _plain(img)
            if not isinstance(img, torch.Tensor) or img.dim() not in (4, 5):
                raise ValueError("augment: image (N, C, D, H, W), (C, D, H, W) or a list of (C, D, H, W), got %r"
                                 % (getattr(img, "shape", img),))
            imgs = list(img) if img.dim() == 5 else [img]
        if not imgs:
            raise ValueError("augment: an empty batch")
        for t in imgs:
            _need_cuda(t, "augment.Compose")
            if t.dtype != torch.float32:
                raise NotImplementedError("augment: the image must be fp32, got %s" % t.dtype)
            if t.dim() != 4 or t.shape[0] != imgs[0].shape[0] or t.device != imgs[0].device:
                raise ValueError("augment: every sample (C, D, H, W) with the same C on one device; got %s"
                                 % [tuple(x.shape) for x in imgs])
        labs = None
        if "label" in self.spatial_keys:
            lab = data["label"]
            if isinstance(lab, (list, tuple)) != listed:
                raise ValueError("augment: the label must take the image's form (a batch or a list)")
            labs = [_plain(t) for t in lab] if listed else (list(_plain(lab)) if _plain(lab).dim() == 5 else [_plain(lab)])
            if len(labs) != len(imgs):
                raise ValueError("augment: %d labels for %d images" % (len(labs), len(imgs)))
            for t, x in zip(labs, imgs):
                _need_cuda(t, "augment.Compose")
                if t.dtype != torch.uint8:
                    raise NotImplementedError("augment: the label must be uint8 (one-hot or label map), got %s" % t.dtype)
                if t.dim() != 4 or t.shape[0] != labs[0].shape[0] or t.shape[1:] != x.shape[1:] or t.device != x.device:
                    raise ValueError("augment: label shape %s does not match image shape %s" % (tuple(t.shape), tuple(x.shape)))
        batched = listed or img.dim() == 5
        return [t.contiguous() for t in imgs], None if labs is None else [t.contiguous() for t in labs], batched

    def _call_geometry(self, data):
        imgs, labs, batched = self._samples(data)
        n, c = len(imgs), imgs[0].shape[0]
        nl = labs[0].shape[0] if labs is not None else 0
        out_size = self.resize.spatial_size
        sizes = [int(np.prod(t.shape[1:])) for t in imgs]
        if max(sizes) >= 1 << 31:
            raise ValueError("augment: every sample fewer than 2^31 voxels per channel, got %d" % max(sizes))
        dev_ = imgs[0].device
        params = self.draw(n, c, out_size)
        crop = self.crop
        pct = crop.percentile if crop is not None else None
        # one pinned upload: int64 sample rows [n][5] and ranks [n][c][2], fp64 affine [n][12], fp32 coef [n][c][2] and gamma [n][c]
        n64, nd, nf = n * 5 + n * c * 2, n * 12, n * c * 3
        host = torch.empty(8 * (n64 + nd) + 4 * nf, dtype=torch.uint8, pin_memory=True)
        h64 = host[: 8 * n64].view(torch.int64)
        h64[: n * 5] = torch.tensor([[x.data_ptr(), labs[i].data_ptr() if labs is not None else 0] + list(x.shape[1:])
                                     for i, x in enumerate(imgs)], dtype=torch.int64).reshape(-1)
        hf = host[8 * (n64 + nd):].view(torch.float32)
        hf[: n * c * 2] = params["coef"].reshape(-1)
        if pct is not None:
            idx = [percentile_index(sz, pct) for sz in sizes]
            h64[n * 5:] = torch.tensor([[lo, hi] * c for lo, hi, _ in idx], dtype=torch.int64).reshape(-1)
            hf[n * c * 2:] = torch.tensor([[float(g)] * c for _, _, g in idx], dtype=torch.float32).reshape(-1)
        host[8 * n64: 8 * (n64 + nd)].view(torch.float64)[:] = params["affine"].reshape(-1)
        dev = host.to(dev_, non_blocking=True)
        d64 = dev[: 8 * n64].view(torch.int64)
        df = dev[8 * (n64 + nd):].view(torch.float32)
        out = torch.empty((n, c) + out_size, dtype=torch.float32, device=dev_)
        lout = torch.empty((n, nl) + out_size, dtype=torch.uint8, device=dev_) if labs is not None else None
        affine = torch.empty(n * 12, dtype=torch.float32, device=dev_)
        box = torch.empty((n, 3, 2), dtype=torch.int32, device=dev_)
        empty = torch.empty(n, dtype=torch.int32, device=dev_)
        thr = torch.empty((n, c), dtype=torch.float32, device=dev_) if pct is not None else None
        norm = self.normalize
        s_out = int(np.prod(out_size))
        with torch.cuda.device(dev_):
            lib = _lib.load_library()
            abytes = int(lib.b200unet_augment_scratch_bytes(n, c, s_out))
            fbytes = int(lib.b200unet_foreground_scratch_bytes(n, c))
            if abytes == 0 or fbytes == 0:
                raise ValueError("augment: %s" % lib.b200unet_last_error().decode())
            scratch = torch.empty(abytes + fbytes, dtype=torch.uint8, device=dev_)
            stream = _lib.stream_ptr()
            _lib.check(lib.b200unet_foreground_box(d64.data_ptr(), n, c, max(sizes), int(crop is not None),
                                                   d64.data_ptr() + 8 * n * 5 if pct is not None else None,
                                                   df.data_ptr() + 4 * n * c * 2 if pct is not None else None,
                                                   crop.margin if crop is not None else 0,
                                                   int(crop.allow_smaller) if crop is not None else 1,
                                                   dev.data_ptr() + 8 * n64, *out_size, affine.data_ptr(), box.data_ptr(),
                                                   empty.data_ptr(), thr.data_ptr() if thr is not None else None,
                                                   scratch.data_ptr() + abytes, stream), "foreground_box")
            _lib.check(lib.b200unet_augment_resample_samples(d64.data_ptr(), n, c, nl, *out_size, affine.data_ptr(),
                                                             _PADDING[self.padding_mode], int(norm is not None and norm.nonzero),
                                                             out.data_ptr(), lout.data_ptr() if lout is not None else None,
                                                             scratch.data_ptr(), stream), "augment_resample_samples")
            if norm is not None or self.intensity:
                _lib.check(lib.b200unet_augment_intensity(out.data_ptr(), n, c, s_out, int(norm is not None),
                                                          int(norm is not None and norm.nonzero),
                                                          int(norm is not None and norm.channel_wise), df.data_ptr(),
                                                          scratch.data_ptr(), stream), "augment_intensity")
        params.update({"box": box, "empty": empty, "threshold": thr, "spatial_size": out_size,
                       "source_affine": affine.view(n, 3, 4)})
        self.last_params = params
        self.last_stats = scratch[: 8 * 3 * n * c].view(torch.float64).view(n, c, 3) if norm is not None else None
        res = dict(data)
        res["image"] = out if batched else out[0]
        if lout is not None:
            res["label"] = lout if batched else lout[0]
        return res


def _make(aug: dict, keys) -> _Transform:
    name = aug["name"]
    if name not in _BY_NAME:
        raise NotImplementedError("augment: transform %r has no device implementation (available: %s)" % (name, sorted(_BY_NAME)))
    return _BY_NAME[name](keys=keys, **{k: v for k, v in aug.items() if k != "name"})


_NORMALIZATIONS = ("zero_mean", "NormalizeIntensity", "NormalizeIntensityd", "NormalizeIntensityD")


_GEOMETRY = ("crop_foreground", "foreground_percentile", "desired_shape", "resample")


def _geometry_transforms(cfg: dict, training: dict) -> list:
    """The training split's crop and resize (``segmentation.py:55-70``, its defaults) as device transforms"""
    def get(key, default):
        return training[key] if key in training else cfg.get(key, default)

    keys, out = ("image", "label"), []
    shape = get("desired_shape", None)
    if get("crop_foreground", False):
        if not shape:
            raise NotImplementedError("augment: crop_foreground without desired_shape gives samples of different sizes; the device "
                                      "stage stacks the batch at desired_shape")
        out.append(CropForegroundd(keys, source_key="image", foreground_percentile=get("foreground_percentile", 0.1), margin=1))
    if shape:
        if get("random_crop", False):
            raise NotImplementedError("augment: random_crop (RandSpatialCropD) has no device implementation")
        if not get("resample", False):
            raise NotImplementedError("augment: desired_shape with resample=False (ResizeWithPadOrCropD) has no device "
                                      "implementation")
        out.append(Resized(keys, spatial_size=shape, mode=("trilinear", "nearest")))
    return out


def build_device_transform(dataset_config: dict, geometry: bool = False):
    """The device ``Compose`` of a config's ``dataset`` section (``training.spatial_augmentations``, ``normalization`` +
    ``normalization_kwargs``, ``training.intensity_augmentations``, read as ``segmentation.py:72-94`` reads them), and a copy of
    the section rewritten so that only the TRAINING dataset leaves that work to the device.  Returns ``(compose, dataset)``.

    ``build_data_loaders`` (``unet3d/scripts/script_utils.py:107-142``) passes the top-level entries to the training AND the
    validation dataset, and the inference loaders read the top level plus ``validation``.  So the top-level ``normalization``
    and ``normalization_kwargs`` move into ``validation`` (entries it already has win), ``training`` gets
    ``normalization=None`` and loses its augmentations: the training dataset then only loads, crops and resizes, while
    validation and inference keep the host z-score the device applies to training batches.  Neither key stays at the top
    level, where it would clash with the per-split entries.

    ``geometry=True`` also moves the training split's ``crop_foreground`` (with ``foreground_percentile``, default 0.1) and
    ``desired_shape`` with ``resample=True`` into the ``Compose`` (``CropForegroundd`` + ``Resized`` ahead of the spatial
    transforms), by the same rule: those four keys move from the top level into ``validation`` and ``training`` gets
    ``crop_foreground=False, desired_shape=None``, so the training dataset only loads, reorients and one-hots; its items
    differ in size, so its loader needs ``collate_fn=list_collate``.  ``random_crop`` and ``desired_shape`` without
    ``resample`` raise ``NotImplementedError``."""
    cfg = copy.deepcopy(dataset_config)
    training = cfg.get("training") or {}
    transforms = _geometry_transforms(cfg, training) if geometry else []
    transforms += [_make(a, ("image", "label")) for a in training.pop("spatial_augmentations", None) or []]
    norm = cfg.get("normalization", "zero_mean")
    if norm is not None:
        if norm not in _NORMALIZATIONS:
            raise NotImplementedError("augment: normalization %r has no device implementation" % (norm,))
        transforms.append(NormalizeIntensityd(keys=("image",), **(cfg.get("normalization_kwargs") or {})))
    transforms += [_make(a, ("image",)) for a in training.pop("intensity_augmentations", None) or []]
    validation = cfg.get("validation") or {}
    for key in ("normalization", "normalization_kwargs") + (_GEOMETRY if geometry else ()):
        if key in cfg:
            validation.setdefault(key, cfg.pop(key))
    training["normalization"] = None
    training.pop("normalization_kwargs", None)
    if geometry:
        for key in _GEOMETRY:
            training.pop(key, None)
        training.update(crop_foreground=False, desired_shape=None)
    cfg["training"] = training
    if validation:
        cfg["validation"] = validation
    return Compose(transforms), cfg
