"""Inference mirror: sliding-window inferer + ``volumetric_predictions`` calling contract.

Reference call sites: /root/reference/unet3d/predict/volumetric.py:131-177 (no_grad loop, ``inferer(x, model)`` or
``model(x)``, activation), unet3d/scripts/script_utils.py:290-293 (``monai.inferers.<name>(**kw)``).  MONAI and
nibabel are absent from this image, so the inferer is restated here (tiles gathered / accumulated on the device)
and file output goes through a caller-supplied ``writer`` instead of ``monai.data.NibabelWriter``.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Callable, List, Optional, Sequence

import numpy as np
import torch

from . import lib as _lib
from . import prepost as _prepost


def _scan_starts(size: int, roi: int, overlap: float) -> List[int]:
    interval = max(int(roi * (1 - overlap)), 1)
    if size <= roi:
        return [0]
    n = int(math.ceil(float(size - roi) / interval)) + 1
    return [min(i * interval, size - roi) for i in range(n)]


def _gaussian_importance(roi: Sequence[int], device, sigma_scale: float = 0.125) -> torch.Tensor:
    w = None
    for r in roi:
        c = (r - 1) / 2.0
        s = sigma_scale * r
        g = torch.exp(-0.5 * ((torch.arange(r, dtype=torch.float32, device=device) - c) / s) ** 2)
        w = g if w is None else w[..., None] * g
    w = w / w.max()
    return torch.clamp(w, min=float(w[w > 0].min()))


class SlidingWindowInferer:
    """``monai.inferers.SlidingWindowInferer(roi_size, sw_batch_size, overlap, mode)`` restated (parity unpinned:
    MONAI is absent from this image).  Tiling runs on the device through libb200unet: one gather kernel per tile batch
    (volume -> [sw_batch, C, roi] NCDHW), the network, one importance-weighted scatter-accumulate kernel (tile order,
    no atomics: deterministic), and a final normalisation by the precomputed weight sum of the scan."""

    def __init__(self, roi_size, sw_batch_size: int = 1, overlap: float = 0.25, mode: str = "constant", **unused):
        self.roi_size = tuple(int(r) for r in (roi_size if hasattr(roi_size, "__len__") else (roi_size,) * 3))
        self.sw_batch_size = int(sw_batch_size)
        if not 1 <= self.sw_batch_size <= 16:
            raise ValueError("sw_batch_size must be in 1..16")
        self.overlap = float(overlap)
        if mode not in ("constant", "gaussian"):
            raise ValueError("mode must be 'constant' or 'gaussian'")
        self.mode = mode
        self._cache = {}

    def _scan(self, shape, device):
        """(roi, importance map, per-axis start lists, weight-sum volume) for this volume shape; cached."""
        key = (tuple(shape), str(device))
        hit = self._cache.get(key)
        if hit is not None:
            return hit
        D, H, W = shape
        roi = [min(r, s) for r, s in zip(self.roi_size, (D, H, W))]
        imp = (torch.ones(roi, device=device) if self.mode == "constant" else _gaussian_importance(roi, device)).contiguous()
        axes = [_scan_starts(s, r, self.overlap) for s, r in zip((D, H, W), roi)]
        dev_axes = [torch.tensor(a, dtype=torch.int32, device=device) for a in axes]
        cnt = torch.empty((D, H, W), dtype=torch.float32, device=device)
        lib = _lib.load_library()
        with torch.cuda.device(device):
            _lib.check(lib.b200unet_tiles_count(dev_axes[0].data_ptr(), len(axes[0]), dev_axes[1].data_ptr(), len(axes[1]),
                                                dev_axes[2].data_ptr(), len(axes[2]), roi[0], roi[1], roi[2], imp.data_ptr(),
                                                cnt.data_ptr(), D, H, W, _lib.stream_ptr()), "tiles_count")
        self._cache = {key: (roi, imp, axes, cnt)}
        return self._cache[key]

    def __call__(self, inputs: torch.Tensor, network: Callable, *args, **kwargs) -> torch.Tensor:
        if not inputs.is_cuda:
            raise RuntimeError("SlidingWindowInferer tiles on the device (no CPU fallback); got %s" % inputs.device)
        x = inputs.as_subclass(torch.Tensor) if type(inputs) is not torch.Tensor else inputs
        x = x.detach().contiguous().float()
        n, c, D, H, W = x.shape
        dev = x.device
        roi, imp, axes, cnt = self._scan((D, H, W), dev)
        jobs = [(b, d, h, w) for b in range(n) for d in axes[0] for h in axes[1] for w in axes[2]]
        lib = _lib.load_library()
        B = self.sw_batch_size
        tiles = torch.empty((B, c) + tuple(roi), dtype=torch.float32, device=dev)
        out = None
        with torch.cuda.device(dev):
            for j0 in range(0, len(jobs), B):
                chunk = jobs[j0:j0 + B]
                padded = chunk + [chunk[-1]] * (B - len(chunk))    # the plan sees a constant batch of sw_batch_size
                starts = (C.c_int32 * (4 * B))(*[v for job in padded for v in job])
                _lib.check(lib.b200unet_tiles_gather(x.data_ptr(), n, c, D, H, W, starts, B, roi[0], roi[1], roi[2],
                                                     tiles.data_ptr(), _lib.stream_ptr()), "tiles_gather")
                pred = network(tiles, *args, **kwargs)
                pred = pred.as_subclass(torch.Tensor) if type(pred) is not torch.Tensor else pred
                if pred.requires_grad:
                    raise RuntimeError("SlidingWindowInferer is inference-only (the reference uses it under torch.no_grad(): "
                                       "training_utils.py:115-147, volumetric.py:140-148); call it inside torch.no_grad()")
                pred = pred.contiguous().float()
                if out is None:
                    out = torch.zeros((n, pred.shape[1], D, H, W), dtype=torch.float32, device=dev)
                starts = (C.c_int32 * (4 * len(chunk)))(*[v for job in chunk for v in job])
                _lib.check(lib.b200unet_tiles_scatter(pred.data_ptr(), pred.shape[1], starts, len(chunk), roi[0], roi[1], roi[2],
                                                      imp.data_ptr(), out.data_ptr(), n, D, H, W, _lib.stream_ptr()),
                           "tiles_scatter")
            _lib.check(lib.b200unet_tiles_normalize(out.data_ptr(), cnt.data_ptr(), n * out.shape[1], D * H * W,
                                                    _lib.stream_ptr()), "tiles_normalize")
        return out


_INFERERS = {"SlidingWindowInferer": SlidingWindowInferer}


def build_inferer_from_config(config):
    """script_utils.py:290-293."""
    kw = dict(config)
    name = kw.pop("name")
    if name not in _INFERERS:
        raise ValueError("inferer {} not supported".format(name))
    return _INFERERS[name](**kw)


def _filename_of(x, index: int):
    """volumetric.py:11-51 semantics: inputs must carry ``meta['filename_or_obj']``."""
    meta = getattr(x, "meta", None)
    if meta is None:
        raise TypeError("volumetric_predictions requires inputs with a 'meta' attribute (MetaTensor-like)")
    if "filename_or_obj" not in meta:
        raise KeyError("filename_or_obj")
    f = meta["filename_or_obj"]
    return f[index] if isinstance(f, (list, tuple)) else f


def _grid_meta_of(x, key: str, index: int, item_ndim: int) -> np.ndarray:
    """``meta[key]`` of item ``index`` as fp64: batched by the collate function (a tensor or array with a leading batch axis),
    a per-item sequence, or one value for every item (``item_ndim`` axes)"""
    meta = x.meta
    if key not in meta:
        raise KeyError("volumetric_predictions(resample=True) needs meta[%r] of the input (LoadImageD records it when it loads "
                       "the image; keep it through the transforms)" % key)
    v = meta[key]
    if isinstance(v, (list, tuple)) and len(v) and np.ndim(_numpy(v[0])) == item_ndim:
        v = v[index]
    v = _numpy(v)
    return v[index] if v.ndim == item_ndim + 1 else v


def _numpy(v) -> np.ndarray:
    if isinstance(v, torch.Tensor):
        return v.as_subclass(torch.Tensor).detach().cpu().double().numpy()
    return np.asarray(v, dtype=np.float64)


def volumetric_predictions(model, dataloader, prediction_dir, activation=None, resample=False, interpolation="trilinear",
                           inferer=None, writer: Optional[Callable] = None):
    """volumetric.py:131-177 without the NIfTI side: returns [(filename, prediction tensor)] and calls
    ``writer(filename, tensor, prediction_dir)`` per item when given.

    ``resample=True`` maps each activated prediction back onto the grid of the image file it came from, as the reference's
    ``ResampleToMatch(mode=interpolation)`` against the re-loaded image: ``prepost.resample_to_match`` from the prediction's grid
    (``meta["affine"]``, the input's affine after orientation, crop and resize) to the file's grid (``meta["original_affine"]``,
    ``meta["spatial_shape"]``, as LoadImageD records them), so the prediction is fp32 ``[C, *spatial_shape]``.  The file is
    not read again."""
    if resample:
        _prepost.resample_mode(interpolation)       # an unsupported mode fails before the model runs
    results = []
    with torch.no_grad():
        for item in dataloader:
            x = item["image"]
            filenames = [_filename_of(x, i) for i in range(x.shape[0])]
            grids = [[_grid_meta_of(x, k, i, nd) for k, nd in (("affine", 2), ("original_affine", 2), ("spatial_shape", 1))]
                     for i in range(x.shape[0])] if resample else None
            xd = x.to(next(model.parameters()).device)
            predictions = inferer(xd, model) if inferer is not None else model(xd)
            if activation == "sigmoid":
                predictions = torch.sigmoid(predictions)
            elif activation == "softmax":
                predictions = torch.softmax(predictions, dim=1)
            elif activation is not None:
                predictions = getattr(torch, activation)(predictions)
            for i, fn in enumerate(filenames):
                p = predictions[i]
                if resample:
                    p = _prepost.resample_to_match(p, *grids[i], mode=interpolation)
                results.append((fn, p))
                if writer is not None:
                    writer(fn, p, prediction_dir)
    return results
