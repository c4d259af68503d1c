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


# MONAI exports both spellings; the reference's configs use the "D" one
RandFlipD, RandRotateD, NormalizeIntensityD = RandFlipd, RandRotated, NormalizeIntensityd
RandScaleIntensityD, RandShiftIntensityD = RandScaleIntensityd, RandShiftIntensityd
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
    plain tensors of the same shapes and dtypes; other entries pass through."""

    def __init__(self, transforms):
        self.transforms = list(transforms)
        stage = {"spatial": 0, "normalize": 1, "intensity": 2}
        last = 0
        for t in self.transforms:
            if not isinstance(t, _Transform):
                raise ValueError("Compose: %r is not a device transform of this module" % (t,))
            s = stage[t.kind]
            if s < last or (s == 1 and last == 1):
                raise ValueError("Compose: the order is spatial transforms, at most one NormalizeIntensityd, then intensity "
                                 "transforms; got %s" % [type(x).__name__ for x in self.transforms])
            last = s
            if t.kind != "spatial" and t.keys != ("image",):
                raise ValueError("%s: keys must be ('image',), got %r" % (type(t).__name__, t.keys))
        self.spatial = [t for t in self.transforms if t.kind == "spatial"]
        self.intensity = [t for t in self.transforms if t.kind == "intensity"]
        norms = [t for t in self.transforms if t.kind == "normalize"]
        self.normalize = norms[0] if norms else None
        keys = {t.keys for t in self.spatial}
        if len(keys) > 1 or not keys <= set(_SPATIAL_KEYS):
            raise ValueError("Compose: every spatial transform takes keys ('image',) or ('image', 'label'), all the same; got %s"
                             % sorted(keys))
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
                if t.kind == "normalize":
                    rec.append({"name": "NormalizeIntensityd", "do": True})
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


def _make(aug: dict, keys) -> _Transform:
    name = aug["name"]
    if name not in _BY_NAME:
        raise NotImplementedError("augment: transform %r has no device implementation (available: %s)" % (name, sorted(_BY_NAME)))
    return _BY_NAME[name](keys=keys, **{k: v for k, v in aug.items() if k != "name"})


_NORMALIZATIONS = ("zero_mean", "NormalizeIntensity", "NormalizeIntensityd", "NormalizeIntensityD")


def build_device_transform(dataset_config: dict):
    """The device ``Compose`` of a config's ``dataset`` section (``training.spatial_augmentations``, ``normalization`` +
    ``normalization_kwargs``, ``training.intensity_augmentations``, read as ``segmentation.py:72-94`` reads them), and a copy of
    the section rewritten so that only the TRAINING dataset leaves that work to the device.  Returns ``(compose, dataset)``.

    ``build_data_loaders`` (``unet3d/scripts/script_utils.py:107-142``) passes the top-level entries to the training AND the
    validation dataset, and the inference loaders read the top level plus ``validation``.  So the top-level ``normalization``
    and ``normalization_kwargs`` move into ``validation`` (entries it already has win), ``training`` gets
    ``normalization=None`` and loses its augmentations: the training dataset then only loads, crops and resizes, while
    validation and inference keep the host z-score the device applies to training batches.  Neither key stays at the top
    level, where it would clash with the per-split entries."""
    cfg = copy.deepcopy(dataset_config)
    training = cfg.get("training") or {}
    transforms = [_make(a, ("image", "label")) for a in training.pop("spatial_augmentations", None) or []]
    norm = cfg.get("normalization", "zero_mean")
    if norm is not None:
        if norm not in _NORMALIZATIONS:
            raise NotImplementedError("augment: normalization %r has no device implementation" % (norm,))
        transforms.append(NormalizeIntensityd(keys=("image",), **(cfg.get("normalization_kwargs") or {})))
    transforms += [_make(a, ("image",)) for a in training.pop("intensity_augmentations", None) or []]
    validation = cfg.get("validation") or {}
    for key in ("normalization", "normalization_kwargs"):
        if key in cfg:
            validation.setdefault(key, cfg.pop(key))
    training["normalization"] = None
    training.pop("normalization_kwargs", None)
    cfg["training"] = training
    if validation:
        cfg["validation"] = validation
    return Compose(transforms), cfg
